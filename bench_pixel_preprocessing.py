#!/usr/bin/env python
"""bench_pixel_preprocessing.py -- the Atari preprocessing layer of the pixel kinds (oracle/SPEC_PIXEL_PREPROCESSING.md):
the plain env step against the reference's stack (frameskip 4, noop_max 30, episodic_life on breakout_pixels,
clip_rewards), and models.Convolutional trained on breakout_pixels under both.

    python bench_pixel_preprocessing.py [--reps K] [--windows W]

Prints one JSON line with the card's name and power limit and
  * `env_step`: pong and breakout_pixels at N = 4 096 and 8 192 envs, vec.send() on its own buffers, timed as CUDA events
    around replays of a CUDA graph of 100 sends, median (with min and max) of --windows windows; the plain env and the
    reference stack alternate window by window in this process.  An agent step of the stack runs up to 4 game ticks
    (fewer only where a game ends), so `ticks_per_s` counts 4 per agent step.  The bytes per agent step do not change with
    the layer (the 28 224-byte row written, the 21 168 bytes of the previous row's three surviving frames read, 16 bytes of
    state, action, reward and flags: 49 408 B); the share is of the H100 SXM data-sheet 3.35 TB/s;
  * `ppo`: evaluate() + train() agent-steps/s on breakout_pixels with models.Convolutional(framestack=4, flat_size=3136),
    1 024 x 128, 4 minibatches x 4 epochs, cuda_graph=True, the plain env and the reference stack alternating call by call
    in one process after two untimed calls each; median with min and max and the graph states.
Writes nothing to the tree."""
import argparse
import json

import numpy as np
import torch

from bench import gpu_info, ppo_config

HBM_PEAK = 3.35e12                  # H100 SXM data sheet, bytes/s
ROW = 4 * 84 * 84
STEP_BYTES = ROW + 3 * 84 * 84 + 16  # 49 408 per agent-step
SENDS = 100
STACK = {'pong': dict(frameskip=4, noop_max=30, clip_rewards=True),
         'breakout_pixels': dict(frameskip=4, noop_max=30, episodic_life=True, clip_rewards=True)}


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=6, help='timed evaluate() + train() calls per config')
    ap.add_argument('--windows', type=int, default=7, help='timed graph windows per kind, config and size')
    return ap.parse_args()


def env_graph(kind, n, kwargs):
    """A vecenv of `kind` and a CUDA graph of SENDS sends on its own buffers (row t-1 -> row t in place)."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200.environments import ocean
    vec = pvec.make(ocean.env_creator(kind), env_kwargs=kwargs, num_envs=n, backend=pvec.B200.options(exact_infos=False))
    acts = torch.as_tensor(np.random.default_rng(0).integers(0, vec.single_action_space.n, size=n), device='cuda')
    vec.async_reset(1)
    vec.recv()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            vec.send(acts)
            vec.recv()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(SENDS):
            vec.send(acts)
            vec.recv()
    g.replay()
    torch.cuda.synchronize()
    return vec, g


def env_section(args):
    out = {}
    for kind in ('pong', 'breakout_pixels'):
        for n in (4096, 8192):
            runs = {'plain': env_graph(kind, n, {}), 'stack': env_graph(kind, n, STACK[kind])}
            times = {k: [] for k in runs}
            for _ in range(args.windows):
                for k, (_, g) in runs.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    g.replay()
                    e1.record()
                    torch.cuda.synchronize()
                    times[k].append(e0.elapsed_time(e1) * 1e-3 / SENDS)
            res = dict(num_envs=n, sends_per_window=SENDS, windows=args.windows, statistic='median', stack=STACK[kind])
            for k, ts in times.items():
                t = float(np.median(ts))
                ticks = 4 if k == 'stack' else 1
                res[k] = dict(us_per_agent_step=t * 1e6, us_min_max=[1e6 * min(ts), 1e6 * max(ts)],
                              agent_steps_per_s=n / t, ticks_per_s=ticks * n / t, bytes_per_agent_step=STEP_BYTES,
                              hbm_gb_per_s=n * STEP_BYTES / t / 1e9, share_of_hbm_peak=n * STEP_BYTES / t / HBM_PEAK)
            res['stack_over_plain_time'] = res['stack']['us_per_agent_step'] / res['plain']['us_per_agent_step']
            out[f'{kind}_n{n}'] = res
            for vec, g in runs.values():
                del g
                vec.close()
            torch.cuda.empty_cache()
    return out


def trainer(kwargs, n, h):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    vec = pvec.make(ocean.env_creator('breakout_pixels'), env_kwargs=kwargs, num_envs=n,
                    backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.Convolutional(vec.driver_env, framestack=4, flat_size=3136)
    policy = cleanrl.Policy(net, fused_sample=True, seed=1).cuda()
    return cp.create(ppo_config(n, h, 'cuda', seed=1, cuda_graph=True, env='breakout_pixels'), vec, policy)


def ppo_section(args):
    from pufferlib_b200 import clean_pufferl as cp
    n, h = 1024, 128
    runs = {'plain': trainer({}, n, h), 'stack': trainer(STACK['breakout_pixels'], n, h)}
    for d in runs.values():
        for _ in range(2):
            cp.evaluate(d)
            cp.train(d)
    times = {k: [] for k in runs}
    for _ in range(args.reps):
        for k, d in runs.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            cp.evaluate(d)
            cp.train(d)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e-3)
    out = dict(num_envs=n, horizon=h, minibatches=4, epochs=4, statistic='median', calls=args.reps)
    for k, d in runs.items():
        ts = times[k]
        out[k] = dict(agent_steps_per_s=n * h / float(np.median(ts)), agent_steps_per_s_min_max=[n * h / max(ts), n * h / min(ts)],
                      rollout_graph_state=d.graph_state, train_graph_state=d.train_graph_state,
                      losses_finite=bool(np.isfinite(d.losses.policy_loss) and np.isfinite(d.losses.value_loss)))
        cp.close(d)
    out['stack_over_plain_rate'] = out['stack']['agent_steps_per_s'] / out['plain']['agent_steps_per_s']
    return out


def main():
    args = parse_args()
    torch.cuda.set_device(0)
    line = dict(gpu=gpu_info(0), method='CUDA events around CUDA-graph replays (env step) or around evaluate()/train() calls')
    line['env_step'] = env_section(args)
    line['ppo'] = ppo_section(args)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
