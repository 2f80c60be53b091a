#!/usr/bin/env python
"""bench_pong.py -- models.Convolutional (NatureCNN on pong's (4, 84, 84) uint8 frames, BASELINE.json C4) with its first
layer on pb_conv1_u8_forward / pb_conv1_u8_wgrad against the stock cuDNN sequence.

    python bench_pong.py [--reps K] [--kernel-reps R] [--skip-c4]

Prints one JSON line with the card's name and power limit and
  * `kernels`: at the C4 training minibatch (131 072 rows) and at the rollout step (4 096 rows): the conv1 forward
    (fast: pb_conv1_u8_forward; stock: x.float() / 255, cuDNN conv1, ReLU) and its backward (fast: pb_conv1_u8_wgrad;
    stock: threshold_backward + cuDNN's weight gradient).  CUDA events around replays of a CUDA graph of --kernel-reps
    launches, median of 5 windows, every shape warmed up.  Algorithmic HBM bytes and FLOPs per minibatch are computed
    here from the shapes (the minimum each op must move; conv1 is 2 * 400 * 32 * 256 FLOP per row each way) and the
    share is of the larger of the two bounds at the H100 SXM data-sheet 3.35 TB/s and 495 TFLOP/s dense TF32;
  * `ppo`: evaluate() + train() and train() alone, agent-steps/s, cuda_graph=True, fast_path True vs False: two trainers
    at 1 024 envs x 128 steps alternated in one process (medians, with min and max, of --reps calls), then C4 itself
    (4 096 x 128) with each path alone in a fresh process, with its rollout and update graph states and
    torch.cuda.max_memory_allocated() (an out-of-memory error is reported as that path's result).
Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

from bench import gpu_info, ppo_config

HBM_PEAK = 3.35e12       # H100 SXM data sheet, bytes/s
TF32_PEAK = 495e12       # dense TF32, FLOP/s
ROW, Y_ROW = 4 * 84 * 84, 32 * 400


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=8, help='timed evaluate() + train() calls per trainer')
    ap.add_argument('--kernel-reps', type=int, default=20, help='launches per captured kernel window')
    ap.add_argument('--skip-c4', action='store_true', help='leave out the 4 096 x 128 runs')
    ap.add_argument('--c4-path', choices=('fast', 'stock'), help='run only C4 on this path and print its result')
    return ap.parse_args()


def graph_time(fn, reps, windows=5):
    """Median over `windows` replays of a CUDA graph of `reps` calls of fn, per call (s)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3 / reps)
    del g
    return float(np.median(times)), [min(times), max(times)]


def roofline(seconds, nbytes, flops):
    t_min = max(nbytes / HBM_PEAK, flops / TF32_PEAK)
    return dict(us=seconds * 1e6, bytes=nbytes, flops=flops, bound='hbm' if nbytes / HBM_PEAK >= flops / TF32_PEAK
                else 'tf32', share_of_bound=t_min / seconds)


def kernel_section(args, m):
    from pufferlib_b200 import _native, models
    lib, dev = _native.lib(), torch.device('cuda')
    torch.manual_seed(0)
    conv = models.layer_init(torch.nn.Conv2d(4, 32, 8, stride=4)).to(dev)
    w, b = conv.weight.detach(), conv.bias.detach()
    x = torch.randint(0, 256, (m, 4, 84, 84), dtype=torch.uint8, device=dev)
    y = torch.empty(m, 32, 20, 20, device=dev)
    P = _native.ptr
    flops = 2 * 400 * 32 * 256 * m
    xb, yb, xf = m * ROW, m * Y_ROW * 4, m * ROW * 4

    def fast_fwd():
        _native.check(lib.pb_conv1_u8_forward(P(x), ROW, m, P(w), P(b), P(y), _native.stream_ptr()))

    def stock_fwd():
        torch.relu(F.conv2d(x.float() / 255.0, w, b, stride=4))

    out = dict(rows=m)
    t, mm = graph_time(fast_fwd, args.kernel_reps)
    out['forward_fast'] = dict(roofline(t, xb + yb, flops), min_max_us=[v * 1e6 for v in mm],
                               kernel='k_conv1_fwd')
    t, mm = graph_time(stock_fwd, args.kernel_reps)
    out['forward_stock'] = dict(roofline(t, xb + xf + 2 * xf + xf + yb + 2 * yb, flops), min_max_us=[v * 1e6 for v in mm],
                                ops='float, /255, cuDNN conv, relu')
    if m > 4096:
        dy = torch.randn(m, 32, 20, 20, device=dev)
        fast_fwd()
        dw, db = torch.empty(32, 256, device=dev), torch.empty(32, device=dev)
        ws = torch.empty(lib.pb_conv1_u8_wgrad_workspace_bytes(m), dtype=torch.uint8, device=dev)

        def fast_bwd():
            _native.check(lib.pb_conv1_u8_wgrad(P(x), ROW, m, P(y), P(dy), P(dw), P(db), P(ws), ws.numel(),
                                                _native.stream_ptr()))
        t, mm = graph_time(fast_bwd, args.kernel_reps)
        out['wgrad_fast'] = dict(roofline(t, xb + 2 * yb, flops), min_max_us=[v * 1e6 for v in mm],
                                 kernel='k_conv1_wgrad + 2 x k_reduce_partials')
        del ws
        xs = x.float() / 255.0

        def stock_bwd():
            dz = torch.ops.aten.threshold_backward(dy, y, 0)
            torch.ops.aten.convolution_backward(dz, xs, w, [32], [4, 4], [0, 0], [1, 1], False, [0, 0], 1,
                                                [False, True, True])
        t, mm = graph_time(stock_bwd, args.kernel_reps)
        out['wgrad_stock'] = dict(roofline(t, 3 * yb + xf + yb, flops), min_max_us=[v * 1e6 for v in mm],
                                  ops='threshold_backward, cuDNN weight gradient')
        del xs, dy
    out['speedup_forward'] = out['forward_stock']['us'] / out['forward_fast']['us']
    if 'wgrad_fast' in out:
        out['speedup_wgrad'] = out['wgrad_stock']['us'] / out['wgrad_fast']['us']
    del x, y
    torch.cuda.empty_cache()
    return out


def make_trainer(n, h, fast):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    vec = pvec.make(ocean.env_creator('pong'), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.Convolutional(vec.driver_env)
    net.fast_path = fast
    policy = cleanrl.Policy(net, fused_sample=True, seed=1).cuda()
    return cp.create(ppo_config(n, h, 'cuda', seed=1, cuda_graph=True, env='pong'), vec, policy)


def timed(cp, d, both, train):
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


def summary(steps, both, train):
    return dict(agent_steps_per_s=steps / float(np.median(both)), train_agent_steps_per_s=steps / float(np.median(train)),
                evaluate_train_ms=1e3 * float(np.median(both)), train_ms=1e3 * float(np.median(train)),
                evaluate_train_ms_min_max=[1e3 * min(both), 1e3 * max(both)],
                train_ms_min_max=[1e3 * min(train), 1e3 * max(train)], calls=len(both))


def c4_section(args):
    """C4 with each path in a fresh process of its own.  Runs before this process touches the device: memory this
    process held would be missing from the runs."""
    c4 = dict(num_envs=4096, horizon=128, minibatch_rows=4096 * 128 // 4, statistic='median',
              method='each path in a process of its own (bench_pong.py --c4-path)')
    for k in ('fast', 'stock'):
        cmd = [sys.executable, os.path.abspath(__file__), '--c4-path', k, '--reps', str(args.reps)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        lines = res.stdout.strip().splitlines()
        c4[k] = json.loads(lines[-1]) if res.returncode == 0 and lines else dict(
            result=f'exit code {res.returncode}', stderr=res.stderr.strip().splitlines()[-3:])
    if 'agent_steps_per_s' in c4['fast'] and 'agent_steps_per_s' in c4['stock']:
        c4['speedup_evaluate_train'] = c4['fast']['agent_steps_per_s'] / c4['stock']['agent_steps_per_s']
        c4['speedup_train'] = c4['fast']['train_agent_steps_per_s'] / c4['stock']['train_agent_steps_per_s']
    return c4


def ppo_section(args):
    from pufferlib_b200 import clean_pufferl as cp
    n, h = 1024, 128
    runs = {'stock': make_trainer(n, h, False), 'fast': make_trainer(n, h, True)}
    for d in runs.values():                 # eager call, then capture + first replay of both graphs
        for _ in range(3):
            cp.evaluate(d)
            cp.train(d)
    both, train = {k: [] for k in runs}, {k: [] for k in runs}
    for _ in range(args.reps):
        for k, d in runs.items():
            timed(cp, d, both[k], train[k])
    out = {'alternated': dict(num_envs=n, horizon=h, statistic='median', **{
        k: dict(summary(n * h, both[k], train[k]), train_graph_state=d.train_graph_state, rollout_graph_state=d.graph_state)
        for k, d in runs.items()})}
    a = out['alternated']
    a['speedup_evaluate_train'] = a['fast']['agent_steps_per_s'] / a['stock']['agent_steps_per_s']
    a['speedup_train'] = a['fast']['train_agent_steps_per_s'] / a['stock']['train_agent_steps_per_s']
    for d in runs.values():
        cp.close(d)
    del runs
    torch.cuda.empty_cache()
    return out


def c4_path(args, fast):
    """C4 (4 096 x 128, 4 minibatches of 131 072 rows, 4 epochs) with conv1 on the fast or the stock path, alone in this
    process: two untimed evaluate() + train() calls (eager, then capture), then max(2, reps / 2) timed ones.  The graph
    states say whether the rollout and the update ran captured (-1: capture failed and the call runs eagerly for good);
    an out-of-memory error is the path's result, with the peak allocated until then."""
    from pufferlib_b200 import clean_pufferl as cp
    n, h = 4096, 128
    torch.cuda.reset_peak_memory_stats()
    d = None
    try:
        d = make_trainer(n, h, fast)
        for _ in range(2):
            cp.evaluate(d)
            cp.train(d)
        b_, t_ = [], []
        for _ in range(max(2, args.reps // 2)):
            timed(cp, d, b_, t_)
        return dict(summary(n * h, b_, t_), train_graph_state=d.train_graph_state, rollout_graph_state=d.graph_state,
                    max_memory_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
    except torch.cuda.OutOfMemoryError as e:
        return dict(result='out of memory', max_memory_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30,
                    train_graph_state=getattr(d, 'train_graph_state', None),
                    rollout_graph_state=getattr(d, 'graph_state', None), error=str(e).splitlines()[0])


def main():
    args = parse_args()
    if args.c4_path:
        torch.cuda.set_device(0)
        print(json.dumps(c4_path(args, args.c4_path == 'fast')))
        return
    c4 = None if args.skip_c4 else c4_section(args)
    torch.cuda.set_device(0)
    line = dict(gpu=gpu_info(0), method='CUDA events around CUDA-graph replays (kernels) or around evaluate()/train() calls')
    line['kernels'] = {'c4_minibatch': kernel_section(args, 131072), 'rollout_step': kernel_section(args, 4096)}
    line['ppo'] = ppo_section(args)
    if c4 is not None:
        line['ppo']['c4'] = c4
    print(json.dumps(line))


if __name__ == '__main__':
    main()
