#!/usr/bin/env python
"""bench_breakout_pixels.py -- breakout from pixels: the breakout_pixels env step and models.Convolutional (NatureCNN)
trained on its (4, 84, 84) uint8 frame stacks.

    python bench_breakout_pixels.py [--reps K] [--windows W] [--skip-4096]

Prints one JSON line with the card's name and power limit and
  * `env_step`: at N = 4 096 and 8 192 envs, vec.send() on its own buffers, timed as CUDA events around replays of a
    CUDA graph of 100 sends, median (with min and max) of --windows windows; breakout_pixels and pong (the same ring and
    the same bytes per row: a same-bytes reference) alternate window by window in this process.  Bytes per agent-step
    are the algorithmic minimum: the 28 224-byte row written, the 21 168 bytes of the previous row's three surviving
    frames read, and 16 bytes of state, action, reward and flags (49 408 B); the share is of the H100 SXM data-sheet
    3.35 TB/s;
  * `ppo`: evaluate() + train() agent-steps/s with models.Convolutional(framestack=4, flat_size=3136), 4 minibatches x 4
    epochs, cuda_graph=True, at 1 024 x 128 and at 4 096 x 128 (14.8 GB of rollout frames), each size in a fresh
    process: two untimed calls (eager, then capture), then --reps timed ones; median with min and max, graph states and
    torch.cuda.max_memory_allocated().
Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

from bench import gpu_info, ppo_config

HBM_PEAK = 3.35e12                  # H100 SXM data sheet, bytes/s
ROW = 4 * 84 * 84
STEP_BYTES = ROW + 3 * 84 * 84 + 16  # 49 408 per agent-step
SENDS = 100


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=6, help='timed evaluate() + train() calls per size')
    ap.add_argument('--windows', type=int, default=7, help='timed graph windows per env kind and size')
    ap.add_argument('--skip-4096', action='store_true', help='leave out the 4 096 x 128 training run')
    ap.add_argument('--ppo-size', type=int, help='run only training at this many envs and print its result')
    return ap.parse_args()


def env_graph(kind, n):
    """A vecenv of `kind` and a CUDA graph of SENDS sends on its own buffers (row t-1 -> row t in place)."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200.environments import ocean
    vec = pvec.make(ocean.env_creator(kind), num_envs=n, backend=pvec.B200.options(exact_infos=False))
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
    for n in (4096, 8192):
        runs = {k: env_graph(k, n) for k in ('breakout_pixels', 'pong')}
        times = {k: [] for k in runs}
        for _ in range(args.windows):
            for k, (_, g) in runs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                g.replay()
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e-3 / SENDS)
        res = dict(num_envs=n, sends_per_window=SENDS, windows=args.windows, statistic='median')
        for k, ts in times.items():
            t = float(np.median(ts))
            res[k] = dict(us_per_step=t * 1e6, us_min_max=[1e6 * min(ts), 1e6 * max(ts)],
                          agent_steps_per_s=n / t, bytes_per_agent_step=STEP_BYTES,
                          hbm_gb_per_s=n * STEP_BYTES / t / 1e9, share_of_hbm_peak=n * STEP_BYTES / t / HBM_PEAK)
        res['breakout_pixels_over_pong_time'] = res['breakout_pixels']['us_per_step'] / res['pong']['us_per_step']
        out[f'n{n}'] = res
        for vec, g in runs.values():
            del g
            vec.close()
        torch.cuda.empty_cache()
    return out


def ppo_size(args, n):
    """evaluate() + train() at n envs x 128 steps, alone in this process."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    h = 128
    torch.cuda.reset_peak_memory_stats()
    d = None
    try:
        vec = pvec.make(ocean.env_creator('breakout_pixels'), num_envs=n, backend=pvec.B200.options(exact_infos=False))
        torch.manual_seed(1)
        net = models.Convolutional(vec.driver_env, framestack=4, flat_size=3136)
        policy = cleanrl.Policy(net, fused_sample=True, seed=1).cuda()
        d = cp.create(ppo_config(n, h, 'cuda', seed=1, cuda_graph=True, env='breakout_pixels'), vec, policy)
        for _ in range(2):
            cp.evaluate(d)
            cp.train(d)
        both, train = [], []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            cp.evaluate(d)
            e[1].record()
            cp.train(d)
            e[2].record()
            torch.cuda.synchronize()
            both.append(e[0].elapsed_time(e[2]) * 1e-3)
            train.append(e[1].elapsed_time(e[2]) * 1e-3)
        steps = n * h
        return dict(num_envs=n, horizon=h, minibatches=4, epochs=4, statistic='median', calls=len(both),
                    agent_steps_per_s=steps / float(np.median(both)),
                    agent_steps_per_s_min_max=[steps / max(both), steps / min(both)],
                    evaluate_train_ms=1e3 * float(np.median(both)), train_ms=1e3 * float(np.median(train)),
                    rollout_graph_state=d.graph_state, train_graph_state=d.train_graph_state,
                    losses_finite=bool(np.isfinite(d.losses.policy_loss) and np.isfinite(d.losses.value_loss)),
                    max_memory_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
    except torch.cuda.OutOfMemoryError as e:
        return dict(num_envs=n, result='out of memory', max_memory_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30,
                    error=str(e).splitlines()[0])


def ppo_section(args):
    """Each size in a fresh process, before this process touches the device."""
    out = {}
    for n in (1024,) + (() if args.skip_4096 else (4096,)):
        cmd = [sys.executable, os.path.abspath(__file__), '--ppo-size', str(n), '--reps', str(args.reps)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        lines = res.stdout.strip().splitlines()
        out[f'n{n}x128'] = json.loads(lines[-1]) if res.returncode == 0 and lines else dict(
            result=f'exit code {res.returncode}', stderr=res.stderr.strip().splitlines()[-3:])
    return out


def main():
    args = parse_args()
    if args.ppo_size:
        torch.cuda.set_device(0)
        print(json.dumps(ppo_size(args, args.ppo_size)))
        return
    ppo = ppo_section(args)
    torch.cuda.set_device(0)
    line = dict(gpu=gpu_info(0), method='CUDA events around CUDA-graph replays (env step) or around evaluate()/train() calls')
    line['env_step'] = env_section(args)
    line['ppo'] = ppo
    print(json.dumps(line))


if __name__ == '__main__':
    main()
