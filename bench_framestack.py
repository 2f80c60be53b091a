#!/usr/bin/env python
"""bench_framestack.py -- one-frame observations (framestack=1) against today's four-frame stack (framestack=4) on the
pixel kinds, at three levels:
  * `env_step`: the env step of pong and breakout_pixels at 4 096 and 8 192 envs, S = 1 and S = 4 alternated window by
    window in one process (CUDA events around replays of a graph of sends), with the share of 3.35 TB/s HBM3 of each
    step's algorithmic bytes (S = 1: 7 056 B written + 16 B of per-row scalars = 7 072 B; S = 4: 21 168 B read +
    28 224 B written + 16 B = 49 408 B);
  * `conv1`: the conv1 kernels (pb_conv1_u8_forward_ex / _wgrad_ex) at 131 072 and 4 096 rows, C = 1 against C = 4, with
    their byte and TF32 FLOP bounds;
  * `ppo`: RecurrentPolicy(LSTMWrapper(Convolutional(framestack=S), 512, 512)) on pong and breakout_pixels, bptt 16,
    4 minibatches x 4 epochs, cuda_graph=True (bench.ppo_config): evaluate() + train() and train() alone at 1 024 x 128
    with the two S alternated in one process, and 4 096 x 128 with each S in a fresh process (peak memory, graph states,
    launches per train()).

    python bench_framestack.py [--reps K] [--windows W] [--skip-c4]

Prints one JSON line with the card's name and power limit.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

from bench import gpu_info, ppo_config
from bench_pong import summary, timed

HBM_PEAK = 3.35e12
TF32_PEAK = 495e12
FRAME = 84 * 84
SCALARS = 16                    # reward f32, terminal, truncation, mask, done f32, the env's packed state word and ctr
STEP_BYTES = {1: FRAME + SCALARS, 4: 3 * FRAME + 4 * FRAME + SCALARS}
SENDS = 20
FRAMESTACKS = (1, 4)


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=6, help='timed evaluate() + train() calls per trainer')
    ap.add_argument('--windows', type=int, default=9, help='timed windows per kind, size and S')
    ap.add_argument('--skip-c4', action='store_true')
    ap.add_argument('--c4', nargs=2, metavar=('ENV', 'S'), help='run 4 096 x 128 of ENV at framestack S alone')
    return ap.parse_args()


def median_ms(ts):
    return 1e3 * float(np.median(ts))


# ---- env step ---------------------------------------------------------------------------------------------------------
def env_graph(kind, n, s):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200.environments import ocean
    vec = pvec.make(ocean.env_creator(kind), env_kwargs={'framestack': s}, num_envs=n,
                    backend=pvec.B200.options(exact_infos=False))
    acts = torch.as_tensor(np.random.default_rng(0).integers(0, vec.single_action_space.n, size=n), device='cuda')
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
    for kind in ('pong', 'breakout_pixels'):
        for n in (4096, 8192):
            runs = {s: env_graph(kind, n, s) for s in FRAMESTACKS}
            times = {s: [] for s in runs}
            for _ in range(args.windows):
                for s, (_, g) in runs.items():
                    replay_time(g, times[s])
            res = dict(num_envs=n, sends_per_window=SENDS, windows=args.windows, statistic='median')
            for s, ts in times.items():
                t = float(np.median(ts))
                res[f'S{s}'] = dict(us_per_step=t * 1e6, us_min_max=[1e6 * min(ts), 1e6 * max(ts)],
                                    agent_steps_per_s=n / t, bytes_per_agent_step=STEP_BYTES[s],
                                    share_of_hbm_peak=n * STEP_BYTES[s] / t / HBM_PEAK)
            res['S4_over_S1_time'] = res['S4']['us_per_step'] / res['S1']['us_per_step']
            out[f'{kind}_n{n}'] = res
            for vec, g in runs.values():
                del g
                vec.close()
            torch.cuda.empty_cache()
    return out


# ---- conv1 kernels ----------------------------------------------------------------------------------------------------
def conv1_section(args):
    from pufferlib_b200 import _native
    lib, P = _native.lib(), _native.ptr
    out = {}
    for m in (131072, 4096):
        res = dict(rows=m, windows=args.windows, statistic='median')
        bufs = {}
        for c in FRAMESTACKS:
            x = torch.randint(0, 256, (m, c, 84, 84), dtype=torch.uint8, device='cuda')
            w = torch.randn(32, 64 * c, device='cuda') * 0.05
            b = torch.zeros(32, device='cuda')
            y = torch.empty(m, 32, 20, 20, device='cuda')
            dy = torch.randn(m, 32, 20, 20, device='cuda')
            dw, db = torch.empty(32, 64 * c, device='cuda'), torch.empty(32, device='cuda')
            ws = torch.empty(lib.pb_conv1_u8_wgrad_workspace_bytes(m), dtype=torch.uint8, device='cuda')
            bufs[c] = (x, w, b, y, dy, dw, db, ws)

        def fwd(c):
            x, w, b, y = bufs[c][:4]
            _native.check(lib.pb_conv1_u8_forward_ex(c, P(x), c * FRAME, m, P(w), P(b), P(y), _native.stream_ptr()))

        def wg(c):
            x, _, _, y, dy, dw, db, ws = bufs[c]
            _native.check(lib.pb_conv1_u8_wgrad_ex(c, P(x), c * FRAME, m, P(y), P(dy), P(dw), P(db), P(ws), ws.numel(),
                                                   _native.stream_ptr()))
        reps = 5 if m > 10000 else 50
        times = {(op, c): [] for op in ('forward', 'wgrad') for c in FRAMESTACKS}
        for op, fn in (('forward', fwd), ('wgrad', wg)):
            for c in FRAMESTACKS:
                fn(c)
        torch.cuda.synchronize()
        for _ in range(args.windows):
            for op, fn in (('forward', fwd), ('wgrad', wg)):
                for c in FRAMESTACKS:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        fn(c)
                    e1.record()
                    torch.cuda.synchronize()
                    times[(op, c)].append(e0.elapsed_time(e1) * 1e-3 / reps)
        for (op, c), ts in times.items():
            t = float(np.median(ts))
            flops = 2.0 * m * 400 * 32 * 64 * c
            x_bytes, y_bytes = m * c * FRAME, m * 32 * 400 * 4
            nbytes = x_bytes + y_bytes if op == 'forward' else x_bytes + 2 * y_bytes
            bound = max(flops / TF32_PEAK, nbytes / HBM_PEAK)
            res[f'{op}_C{c}'] = dict(ms=1e3 * t, ms_min_max=[1e3 * min(ts), 1e3 * max(ts)], flops=flops, bytes=nbytes,
                                     bound_ms=1e3 * bound, bound_by='bytes' if nbytes / HBM_PEAK > flops / TF32_PEAK
                                     else 'tf32', share_of_bound=bound / t)
        for op in ('forward', 'wgrad'):
            res[f'{op}_C4_over_C1_time'] = res[f'{op}_C4']['ms'] / res[f'{op}_C1']['ms']
        out[f'm{m}'] = res
        del bufs
        torch.cuda.empty_cache()
    return out


# ---- PPO with the Atari LSTM policy -----------------------------------------------------------------------------------
def make_trainer(env, n, h, s):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    vec = pvec.make(ocean.env_creator(env), env_kwargs={'framestack': s}, num_envs=n,
                    backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.LSTMWrapper(vec.driver_env, models.Convolutional(vec.driver_env, framestack=s), input_size=512,
                             hidden_size=512)
    policy = cleanrl.RecurrentPolicy(net, seed=1).cuda()
    cfg = ppo_config(n, h, 'cuda', seed=1, cuda_graph=True, env=env)
    cfg.fused_loss = True
    return cp.create(cfg, vec, policy)


def states(d):
    return dict(train_graph_state=d.train_graph_state, rollout_graph_state=d.graph_state,
                minibatch_path=d.train_minibatch_path, msg=d.msg or None)


def alternated(args, env):
    from pufferlib_b200 import clean_pufferl as cp
    n, h = 1024, 128
    runs = {s: make_trainer(env, n, h, s) for s in FRAMESTACKS}
    for d in runs.values():
        for _ in range(3):
            cp.evaluate(d)
            cp.train(d)
    both, train = {s: [] for s in runs}, {s: [] for s in runs}
    for _ in range(args.reps):
        for s, d in runs.items():
            timed(cp, d, both[s], train[s])
    a = dict(num_envs=n, horizon=h, statistic='median', **{
        f'S{s}': dict(summary(n * h, both[s], train[s]), **states(d)) for s, d in runs.items()})
    a['S1_over_S4_rate'] = a['S1']['agent_steps_per_s'] / a['S4']['agent_steps_per_s']
    a['S1_over_S4_train_rate'] = a['S1']['train_agent_steps_per_s'] / a['S4']['train_agent_steps_per_s']
    for d in runs.values():
        cp.close(d)
    del runs
    torch.cuda.empty_cache()
    return a


def c4_run(args, env, s):
    from pufferlib_b200 import _native, clean_pufferl as cp
    n, h = 4096, 128
    torch.cuda.reset_peak_memory_stats()
    d = make_trainer(env, n, h, int(s))
    for _ in range(2):
        cp.evaluate(d)
        cp.train(d)
    lib = _native.lib()
    cp.evaluate(d)
    torch.cuda.synchronize()
    l0 = lib.pb_launch_count()
    cp.train(d)
    torch.cuda.synchronize()
    launches = dict(from_python=int(lib.pb_launch_count() - l0),
                    in_graph=int(d.train_graph_launches) if d.train_graph_state == 2 else 0)
    b_, t_ = [], []
    for _ in range(max(2, args.reps // 2)):
        timed(cp, d, b_, t_)
    return dict(summary(n * h, b_, t_), **states(d), launches_per_train=launches,
                rollout_obs_gib=d.experience.obs.numel() / 2 ** 30,
                max_memory_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def subprocess_json(extra):
    res = subprocess.run([sys.executable, os.path.abspath(__file__)] + extra, capture_output=True, text=True)
    lines = res.stdout.strip().splitlines()
    return json.loads(lines[-1]) if res.returncode == 0 and lines else dict(
        result=f'exit code {res.returncode}', stderr=res.stderr.strip().splitlines()[-3:])


def main():
    args = parse_args()
    if args.c4:
        torch.cuda.set_device(0)
        print(json.dumps(c4_run(args, *args.c4)))
        return
    line = {}
    if not args.skip_c4:       # before this process touches the device
        line['c4'] = {env: {f'S{s}': subprocess_json(['--c4', env, str(s), '--reps', str(args.reps)])
                            for s in FRAMESTACKS} for env in ('pong', 'breakout_pixels')}
    torch.cuda.set_device(0)
    line['gpu'] = gpu_info(0)
    line['method'] = 'CUDA events: around graph replays (env step), kernel loops (conv1), evaluate()/train() calls (ppo)'
    line['env_step'] = env_section(args)
    line['conv1'] = conv1_section(args)
    line['ppo'] = {env: alternated(args, env) for env in ('pong', 'breakout_pixels')}
    print(json.dumps(line))


if __name__ == '__main__':
    main()
