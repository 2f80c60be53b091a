#!/usr/bin/env python
"""bench_pong_versus.py -- two-player pong from pixels (pong_versus, two agent rows per env) against pong, at two
levels:
  * `env_step`: the env step at 4 096 and 8 192 envs (8 192 and 16 384 agent rows), S = 4 and S = 1, alternated window
    by window with pong's step at the same S and the same number of agent rows, in one process (CUDA events around
    replays of a graph of sends).  Per agent step the algorithmic bytes are pong's -- S = 4: 21 168 B read + 28 224 B
    written + 16 B of per-row scalars = 49 408 B; S = 1: 7 056 + 16 = 7 072 B -- and the share of 3.35 TB/s HBM3 is
    given for both kinds;
  * `ppo`: cleanrl.Policy(models.Convolutional(framestack=4)) at 1 024 envs (2 048 agent rows) x 128 steps, bptt 16,
    4 minibatches x 4 epochs, cuda_graph=True (bench.ppo_config): evaluate() + train() agent-steps/s, graph states,
    the update plan and peak memory.

    python bench_pong_versus.py [--reps K] [--windows W]

Prints one JSON line with the card's name and power limit.  Writes nothing to the tree."""
import argparse
import json

import numpy as np
import torch

from bench import gpu_info, ppo_config
from bench_pong import summary, timed

HBM_PEAK = 3.35e12
FRAME = 84 * 84
SCALARS = 16                    # reward f32, terminal, truncation, mask, done f32, the env's packed state words and ctr
STEP_BYTES = {1: FRAME + SCALARS, 4: 3 * FRAME + 4 * FRAME + SCALARS}
SENDS = 20


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=6, help='timed evaluate() + train() calls')
    ap.add_argument('--windows', type=int, default=9, help='timed windows per kind, size and S')
    return ap.parse_args()


def env_graph(kind, n, s):
    """A graph of SENDS sends of `kind` with n envs at framestack s, warmed up."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200.environments import ocean
    vec = pvec.make(ocean.env_creator(kind), env_kwargs={'framestack': s}, num_envs=n,
                    backend=pvec.B200.options(exact_infos=False))
    acts = torch.as_tensor(np.random.default_rng(0).integers(0, 6, size=vec.num_agents), device='cuda')
    vec.async_reset(1)
    vec.recv()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(3):
            vec.send(acts)
            vec.recv()
    torch.cuda.current_stream().wait_stream(st)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(SENDS):
            vec.send(acts)
            vec.recv()
    g.replay()
    torch.cuda.synchronize()
    return vec, g


def replay_time(g, times):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    times.append(e0.elapsed_time(e1) * 1e-3 / SENDS)


def env_section(args):
    out = {}
    for s in (4, 1):
        for n in (4096, 8192):
            rows = 2 * n
            # pong_versus with n envs, pong with as many envs as pong_versus has agent rows
            runs = {'pong_versus': env_graph('pong_versus', n, s), 'pong': env_graph('pong', rows, s)}
            times = {k: [] for k in runs}
            for _ in range(args.windows):
                for k, (_, g) in runs.items():
                    replay_time(g, times[k])
            res = dict(num_envs=n, agent_rows=rows, framestack=s, sends_per_window=SENDS, windows=args.windows,
                       statistic='median', bytes_per_agent_step=STEP_BYTES[s])
            for k, ts in times.items():
                t = float(np.median(ts))
                res[k] = dict(us_per_step=t * 1e6, us_min_max=[1e6 * min(ts), 1e6 * max(ts)],
                              ns_per_agent_step=t * 1e9 / rows, agent_steps_per_s=rows / t,
                              share_of_hbm_peak=rows * STEP_BYTES[s] / t / HBM_PEAK)
            res['versus_over_pong_time'] = res['pong_versus']['us_per_step'] / res['pong']['us_per_step']
            out[f'S{s}_n{n}'] = res
            for vec, g in runs.values():
                del g
                vec.close()
            torch.cuda.empty_cache()
    return out


def ppo_section(args):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    n, h = 1024, 128
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    vec = pvec.make(ocean.env_creator('pong_versus'), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    policy = cleanrl.Policy(models.Convolutional(vec.driver_env), fused_sample=True, seed=1).cuda()
    plans = []
    update_plan = cp.update_plan
    cp.update_plan = lambda d: plans.append(update_plan(d)) or plans[-1]
    try:
        d = cp.create(ppo_config(vec.num_agents, h, 'cuda', seed=1, cuda_graph=True, env='pong_versus'), vec, policy)
        for _ in range(3):
            cp.evaluate(d)
            cp.train(d)
        both, train = [], []
        for _ in range(args.reps):
            timed(cp, d, both, train)
    finally:
        cp.update_plan = update_plan
    torch.cuda.synchronize()
    res = dict(summary(vec.num_agents * h, both, train), num_envs=n, agent_rows=vec.num_agents, horizon=h,
               train_graph_state=d.train_graph_state, rollout_graph_state=d.graph_state,
               plan=[plans[-1].engine, plans[-1].form] if plans else None,
               losses_finite=bool(np.isfinite([d.losses.policy_loss, d.losses.value_loss]).all()),
               max_memory_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
    cp.close(d)
    return res


def main():
    args = parse_args()
    torch.cuda.set_device(0)
    out = dict(bench='pong_versus', gpu=gpu_info(0))
    out['env_step'] = env_section(args)
    out['ppo_convolutional'] = ppo_section(args)
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
