"""Self-play on pong_versus: one cleanrl.Policy(models.Convolutional(framestack=4)) drives both paddles of every env, and
the mean game length in ticks is the learning signal -- rallies lengthen as both seats learn to return the ball, while
the two seats' mean scores stay exact negatives (zero-sum).  Not collected by pytest.

    python tests/experimental/check_pong_versus_selfplay.py [--envs N] [--horizon H] [--iters K] [--max-score S]

Prints one JSON line per logged window of iterations ({iter, agent_steps, rollouts_with_games, episode_length,
score_1, score_2}: means over the window's rollouts of evaluate()'s per-agent means) and a summary line with the card's
name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from bench import gpu_info, ppo_config  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=1024)
    ap.add_argument('--horizon', type=int, default=128)
    ap.add_argument('--iters', type=int, default=60)
    ap.add_argument('--max-score', type=int, default=3)
    ap.add_argument('--log-every', type=int, default=5)
    args = ap.parse_args()

    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl

    torch.cuda.set_device(0)
    vec = pvec.make(ocean.env_creator('pong_versus'), env_kwargs={'max_score': args.max_score}, num_envs=args.envs,
                    backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    policy = cleanrl.Policy(models.Convolutional(vec.driver_env), fused_sample=True, seed=1).cuda()
    d = cp.create(ppo_config(vec.num_agents, args.horizon, 'cuda', seed=1, cuda_graph=True, env='pong_versus'), vec,
                  policy)
    steps, t0, rows, window = 0, time.time(), [], []
    for it in range(1, args.iters + 1):
        stats, _ = cp.evaluate(d)      # the rollout's per-agent means, from the device's agent statistics
        cp.train(d)
        steps += vec.num_agents * args.horizon
        if '1/episode_length' in stats:
            window.append((stats['1/episode_length'], stats['1/score'], stats['2/score']))
        if it % args.log_every == 0:
            w = np.asarray(window) if window else np.full((1, 3), np.nan)
            row = dict(iter=it, agent_steps=steps, rollouts_with_games=len(window),
                       episode_length=float(w[:, 0].mean()), score_1=float(w[:, 1].mean()),
                       score_2=float(w[:, 2].mean()))
            rows.append(row)
            window = []
            print(json.dumps(row), flush=True)
    lengths = [r['episode_length'] for r in rows if np.isfinite(r['episode_length'])]
    print(json.dumps(dict(summary='pong_versus self-play', gpu=gpu_info(0), envs=args.envs, horizon=args.horizon,
                          iters=args.iters, max_score=args.max_score, agent_steps=steps, seconds=time.time() - t0,
                          first_episode_length=lengths[0] if lengths else None,
                          last_episode_length=lengths[-1] if lengths else None,
                          losses_finite=bool(np.isfinite([d.losses.policy_loss, d.losses.value_loss]).all()))),
          flush=True)
    cp.close(d)


if __name__ == '__main__':
    main()
