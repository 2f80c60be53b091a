#!/usr/bin/env python
"""bench_nature_trunk.py -- models.Convolutional's conv2 and conv3 (the NatureCNN trunk after conv1) on
pb_nature_conv_forward / _dgrad / _wgrad against the cuDNN sequence they replace, allow_tf32 on (torch's default).

    python bench_nature_trunk.py [--reps K] [--kernel-reps R] [--skip-c4] [--skip-profile]

Prints one JSON line with the card's name and power limit and
  * `profile`: per-op CUDA time (torch.profiler, in a process of its own) of one C4 minibatch's (131 072 rows) model
    forward + backward from uint8 frames, with the trunk path and with the trunk refused;
  * `kernels`: at 131 072 rows (a C4 minibatch) and 4 096 rows (a rollout step): the forward (both layers: new kernels
    vs cuDNN conv + ReLU) and the backward (both layers' input and weight gradients: new kernels vs threshold_backward +
    cuDNN convolution_backward), CUDA events around replays of a CUDA graph of --kernel-reps calls, median of 5 windows,
    with the minimum HBM bytes and the FLOPs from the shapes and the share of the larger bound at the H100 SXM data
    sheet's 3.35 TB/s and 495 TFLOP/s dense TF32;
  * `ppo`: evaluate() + train() agent-steps/s on pong and breakout_pixels, cuda_graph=True, trunk path vs refused: two
    trainers at 1 024 x 128 alternated in one process, then 4 096 x 128 (C4) with each path alone in a fresh process,
    with peak memory.
Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

from bench import gpu_info, ppo_config
from bench_pong import graph_time, roofline, summary, timed

# layer: x shape, w shape, stride, y shape
LAYERS = {2: ((32, 20, 20), (64, 32, 4, 4), 2, (64, 9, 9)), 3: ((64, 9, 9), (64, 64, 3, 3), 1, (64, 7, 7))}


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=6, help='timed evaluate() + train() calls per trainer')
    ap.add_argument('--kernel-reps', type=int, default=10, help='calls per captured kernel window')
    ap.add_argument('--skip-c4', action='store_true')
    ap.add_argument('--skip-profile', action='store_true')
    ap.add_argument('--c4', nargs=2, metavar=('ENV', 'PATH'), help='run C4 of ENV on PATH (trunk / refused) alone')
    ap.add_argument('--profile-only', action='store_true')
    return ap.parse_args()


def numel(shape):
    return int(np.prod(shape))


def kernel_section(args, m):
    from pufferlib_b200 import _native
    lib, dev, P = _native.lib(), torch.device('cuda'), _native.ptr
    torch.manual_seed(0)
    t = {}
    for layer, (xs, ws, s, ys) in LAYERS.items():
        t[layer] = dict(x=torch.relu(torch.randn(m, *xs, device=dev)), w=torch.randn(*ws, device=dev) * 0.05,
                        b=torch.randn(64, device=dev) * 0.05, y=torch.empty(m, *ys, device=dev),
                        dy=torch.randn(m, *ys, device=dev), dx=torch.empty(m, *xs, device=dev),
                        dw=torch.empty(*ws, device=dev), db=torch.empty(64, device=dev),
                        ws=torch.empty(lib.pb_nature_conv_wgrad_workspace_bytes(layer, m), dtype=torch.uint8, device=dev))
    sp = _native.stream_ptr

    def new_fwd():
        for layer, d in t.items():
            _native.check(lib.pb_nature_conv_forward(layer, P(d['x']), m, P(d['w']), P(d['b']), P(d['y']), sp()))

    def ref_fwd():
        for layer, d in t.items():
            torch.relu(torch.nn.functional.conv2d(d['x'], d['w'], d['b'], stride=LAYERS[layer][2]))

    def new_bwd():
        for layer, d in t.items():
            _native.check(lib.pb_nature_conv_dgrad(layer, P(d['y']), P(d['dy']), P(d['w']), m, P(d['dx']), sp()))
            _native.check(lib.pb_nature_conv_wgrad(layer, P(d['x']), P(d['y']), P(d['dy']), m, P(d['dw']), P(d['db']),
                                                   P(d['ws']), d['ws'].numel(), sp()))

    def ref_bwd():
        for layer, d in t.items():
            s = LAYERS[layer][2]
            dz = torch.ops.aten.threshold_backward(d['dy'], d['y'], 0)
            torch.ops.aten.convolution_backward(dz, d['x'], d['w'], [64], [s, s], [0, 0], [1, 1], False, [0, 0], 1,
                                                [True, True, True])
    new_fwd()
    f32 = 4
    xb = sum(numel(LAYERS[k][0]) for k in LAYERS) * f32 * m
    yb = sum(numel(LAYERS[k][3]) for k in LAYERS) * f32 * m
    ffl = sum(2 * numel(LAYERS[k][3][1:]) * 64 * numel(LAYERS[k][1][1:]) for k in LAYERS) * m
    out = dict(rows=m)
    for name, fn, nbytes, fl in (('forward_new', new_fwd, xb + yb, ffl), ('forward_cudnn', ref_fwd, xb + yb, ffl),
                                 ('backward_new', new_bwd, xb + 2 * yb + xb, 2 * ffl),
                                 ('backward_cudnn', ref_bwd, xb + 2 * yb + xb, 2 * ffl)):
        tm, mm = graph_time(fn, args.kernel_reps)
        out[name] = dict(roofline(tm, nbytes, fl), min_max_us=[v * 1e6 for v in mm])
    out['speedup_forward'] = out['forward_cudnn']['us'] / out['forward_new']['us']
    out['speedup_backward'] = out['backward_cudnn']['us'] / out['backward_new']['us']
    del t
    torch.cuda.empty_cache()
    return out


def fake_env():
    import types
    from pufferlib_b200 import spaces
    return types.SimpleNamespace(single_observation_space=spaces.Box(0, 255, (4, 84, 84), np.uint8),
                                 single_action_space=spaces.Discrete(6))


def profile_section():
    """One C4 minibatch's forward + backward, per-op CUDA time, trunk path vs refused (each after a warm-up call)."""
    from torch.profiler import ProfilerActivity, profile
    from pufferlib_b200 import models
    m = 131072
    x = torch.randint(0, 256, (m, 4, 84, 84), dtype=torch.uint8, device='cuda')
    out = {}
    for path in ('trunk', 'refused'):
        torch.manual_seed(0)
        net = models.Convolutional(fake_env()).cuda()
        if path == 'refused':
            net._trunk_ok = lambda: False

        def step():
            logits, value = net(x)
            (logits.sum() + value.sum()).backward()
        step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        rows = []
        for ev in prof.key_averages():
            us = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0)
            if us > 0 and ev.key and not ev.key.startswith('aten::') and 'Memcpy' not in ev.key:
                rows.append((ev.key[:90], us / 1e3, ev.count))
        rows.sort(key=lambda r: -r[1])
        out[path] = dict(total_ms=sum(r[1] for r in rows), ops=[dict(name=n, ms=t_, calls=c) for n, t_, c in rows[:16]])
        del net
        torch.cuda.empty_cache()
    return out


def make_trainer(env, n, h, trunk):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.Convolutional(vec.driver_env)
    if not trunk:
        net._trunk_ok = lambda: False
    policy = cleanrl.Policy(net, fused_sample=True, seed=1).cuda()
    return cp.create(ppo_config(n, h, 'cuda', seed=1, cuda_graph=True, env=env), vec, policy)


def alternated(args, env):
    from pufferlib_b200 import clean_pufferl as cp
    n, h = 1024, 128
    runs = {'refused': make_trainer(env, n, h, False), 'trunk': make_trainer(env, n, h, True)}
    for d in runs.values():
        for _ in range(3):
            cp.evaluate(d)
            cp.train(d)
    both, train = {k: [] for k in runs}, {k: [] for k in runs}
    for _ in range(args.reps):
        for k, d in runs.items():
            timed(cp, d, both[k], train[k])
    a = dict(num_envs=n, horizon=h, statistic='median', **{
        k: dict(summary(n * h, both[k], train[k]), train_graph_state=d.train_graph_state, rollout_graph_state=d.graph_state)
        for k, d in runs.items()})
    a['speedup_evaluate_train'] = a['trunk']['agent_steps_per_s'] / a['refused']['agent_steps_per_s']
    for d in runs.values():
        cp.close(d)
    del runs
    torch.cuda.empty_cache()
    return a


def c4_run(args, env, trunk):
    from pufferlib_b200 import clean_pufferl as cp
    n, h = 4096, 128
    torch.cuda.reset_peak_memory_stats()
    d = make_trainer(env, n, h, trunk)
    for _ in range(2):
        cp.evaluate(d)
        cp.train(d)
    b_, t_ = [], []
    for _ in range(max(2, args.reps // 2)):
        timed(cp, d, b_, t_)
    return dict(summary(n * h, b_, t_), train_graph_state=d.train_graph_state, rollout_graph_state=d.graph_state,
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
        print(json.dumps(c4_run(args, args.c4[0], args.c4[1] == 'trunk')))
        return
    if args.profile_only:
        torch.cuda.set_device(0)
        print(json.dumps(profile_section()))
        return
    line = {}
    if not args.skip_c4:       # before this process touches the device
        c4 = {}
        for env in ('pong', 'breakout_pixels'):
            c4[env] = {p: subprocess_json(['--c4', env, p, '--reps', str(args.reps)]) for p in ('trunk', 'refused')}
            r = c4[env]
            if 'agent_steps_per_s' in r['trunk'] and 'agent_steps_per_s' in r['refused']:
                r['speedup_evaluate_train'] = r['trunk']['agent_steps_per_s'] / r['refused']['agent_steps_per_s']
        line['c4'] = c4
    if not args.skip_profile:
        line['profile'] = subprocess_json(['--profile-only'])
    torch.cuda.set_device(0)
    line['gpu'] = gpu_info(0)
    line['method'] = 'CUDA events around CUDA-graph replays (kernels) or around evaluate()/train() calls'
    line['kernels'] = {'c4_minibatch': kernel_section(args, 131072), 'rollout_step': kernel_section(args, 4096)}
    line['ppo'] = {env: alternated(args, env) for env in ('pong', 'breakout_pixels')}
    print(json.dumps(line))


if __name__ == '__main__':
    main()
