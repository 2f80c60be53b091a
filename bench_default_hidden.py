#!/usr/bin/env python
"""bench_default_hidden.py -- models.Default with 256 hidden units on the hand-written kernels.

    python bench_default_hidden.py [--num-envs N] [--horizon H] [--hidden 256] [--reps K] [--kernel-reps R]

Prints one JSON line with
  * `breakout`: breakout with Default(hidden_size=--hidden), CUDA-graphed rollout and update, two trainers built the
    same way in one process and alternated: `plain` (fast_path=False, manual_update=False: nn.Linear forward, library
    GEMMs + pb_sample_logits at rollout time, autograd backward, clip_grad_norm_ and torch.optim.Adam, the path these
    models took before the H > 128 kernels) and `kernels` (pb_policy_mlp_sample's chunked rollout step, the
    _DefaultMLPUpdate chain with the sliced pb_mlp_tail_backward_ex).  Agent-steps/s of evaluate() + train() and of
    train() alone (CUDA events around each call, medians of --reps) and the kernels one captured train() replays
    (bench_default_heads.graph_kernels);
  * `policy_step`: pb_policy_mlp_sample at 16 384 rows of 128 features and 4 actions, H = --hidden vs H = 128,
    alternated, CUDA events over --kernel-reps launches, median of 5 windows;
  * `mlp_tail`: pb_mlp_tail_backward_ex at 524 288 rows, 8 head rows, H = --hidden, TMA-staged kernel; algorithmic HBM
    bytes per row 2 * 4H + 4R (hidden read, dPre written) plus 4R per 128-column slice (each slice reads the row's dOut)
    over the time, against the H100 SXM data-sheet 3.35 TB/s.
The card's name and power limit go with the numbers.  Writes nothing to the tree."""
import argparse
import json
import types

import numpy as np
import torch

from bench import gpu_info, ppo_config
from bench_default_heads import HBM_PEAK, alternate, graph_kernels


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-envs', type=int, default=16384)
    ap.add_argument('--horizon', type=int, default=128)
    ap.add_argument('--hidden', type=int, default=256)
    ap.add_argument('--reps', type=int, default=10, help='timed evaluate() + train() calls per trainer')
    ap.add_argument('--kernel-reps', type=int, default=100, help='launches per timed kernel window')
    return ap.parse_args()


def make_trainer(args, kernels):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    n, h = args.num_envs, args.horizon
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.Default(vec.driver_env, hidden_size=args.hidden)
    net.fast_path = kernels
    policy = cleanrl.Policy(net, fused_sample=True, seed=1).cuda()
    cfg = ppo_config(n, h, 'cuda', seed=1, cuda_graph=True, env='breakout')
    cfg.manual_update = kernels
    return cp.create(cfg, vec, policy)


def breakout_section(args):
    from pufferlib_b200 import clean_pufferl as cp
    runs = {'plain': make_trainer(args, False), 'kernels': make_trainer(args, True)}
    for d in runs.values():                 # eager call, then capture + first replay of both graphs
        for _ in range(3):
            cp.evaluate(d)
            cp.train(d)
    steps = args.num_envs * args.horizon
    both, train = {k: [] for k in runs}, {k: [] for k in runs}
    for _ in range(args.reps):
        for k, d in runs.items():
            torch.cuda.synchronize()
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            cp.evaluate(d)
            e[1].record()
            cp.train(d)
            e[2].record()
            torch.cuda.synchronize()
            both[k].append(e[0].elapsed_time(e[2]) * 1e-3)
            train[k].append(e[1].elapsed_time(e[2]) * 1e-3)
    out = {}
    for k, d in runs.items():
        mu = d.manual_update
        out[k] = dict(
            agent_steps_per_s=steps / float(np.median(both[k])), train_agent_steps_per_s=steps / float(np.median(train[k])),
            evaluate_train_ms=1e3 * float(np.median(both[k])), train_ms=1e3 * float(np.median(train[k])),
            evaluate_train_ms_min_max=[1e3 * min(both[k]), 1e3 * max(both[k])],
            train_ms_min_max=[1e3 * min(train[k]), 1e3 * max(train[k])],
            kernels_per_train=graph_kernels(cp, d), project_kernels_in_train_graph=d.train_graph_launches,
            train_graph_state=d.train_graph_state, rollout_graph_state=d.graph_state,
            fused_rollouts=getattr(d, 'fused_rollouts', 0), minibatch_form=d.train_minibatch_path,
            update='hand-written' if mu is not None else 'autograd', used_fused=getattr(mu, 'used_fused', None))
    for d in runs.values():
        cp.close(d)
    out['speedup_evaluate_train'] = out['kernels']['agent_steps_per_s'] / out['plain']['agent_steps_per_s']
    out['speedup_train'] = out['kernels']['train_agent_steps_per_s'] / out['plain']['train_agent_steps_per_s']
    out.update(num_envs=args.num_envs, horizon=args.horizon, hidden=args.hidden, reps=args.reps, statistic='median')
    return out


def policy_section(args, m=16384, n_act=4):
    from pufferlib_b200 import models
    from pufferlib_b200.frameworks import cleanrl
    from pufferlib_b200.spaces import Box, Discrete
    dev = torch.device('cuda')
    env = types.SimpleNamespace(single_observation_space=Box(0, 1, (128,), np.float32), single_action_space=Discrete(n_act))
    x = torch.randn(m, 128, device=dev)
    fns = {}
    for hid in (args.hidden, 128):
        torch.manual_seed(hid)
        pol = cleanrl.Policy(models.Default(env, hidden_size=hid), fused_sample=True, seed=1).to(dev)
        outs = (torch.empty(m, device=dev), torch.empty(m, device=dev), torch.empty(m, dtype=torch.int64, device=dev))
        with torch.no_grad():
            assert pol._policy_step_fused(x, outs) is not None
        fns[f'H{hid}'] = (lambda p=pol, o=outs: p._policy_step_fused(x, o))
    with torch.no_grad():
        t = alternate(fns, args.kernel_reps)
    return dict(rows=m, features=128, n_act=n_act, launches_per_window=args.kernel_reps, windows=5, statistic='median',
                method='CUDA events around back-to-back host calls of Policy._policy_step_fused (one kernel each)',
                **{k: dict(us=v * 1e6) for k, v in t.items()})


def tail_section(args, m=524288, rows=8):
    from pufferlib_b200 import _native
    lib, dev, hid = _native.lib(), torch.device('cuda'), args.hidden
    torch.manual_seed(0)
    hidden = torch.relu(torch.randn(m, hid, device=dev))
    dpre = torch.empty_like(hidden)
    dout = torch.randn(m, rows, device=dev) / m
    w = torch.randn(rows, hid, device=dev)
    grads = torch.empty(rows * hid + hid + rows, device=dev)
    ws = torch.empty(lib.pb_mlp_tail_workspace_bytes_ex(m, hid, rows), dtype=torch.uint8, device=dev)
    a = (_native.ptr(dout), rows, _native.ptr(w), _native.ptr(hidden), m, hid, _native.ptr(dpre), _native.ptr(grads),
         _native.ptr(ws), ws.numel(), rows, _native.stream_ptr())
    t = alternate({'tail': lambda: _native.check(lib.pb_mlp_tail_backward_ex(*a))}, args.kernel_reps)['tail']
    bytes_per_row = 2 * 4 * hid + 4 * rows * (hid // 128)
    bw = bytes_per_row * m / t
    return dict(rows=m, hidden=hid, head_rows=rows, kernel='k_mlp_tail_bwd<8, TMA> + k_reduce_partials',
                bytes_per_row=bytes_per_row, us=t * 1e6, tb_per_s=bw / 1e12, share_of_hbm_peak=bw / HBM_PEAK,
                launches_per_window=args.kernel_reps, windows=5, statistic='median')


def main():
    args = parse_args()
    torch.cuda.set_device(0)
    line = dict(gpu=gpu_info(0))
    line['mlp_tail'] = tail_section(args)
    line['policy_step'] = policy_section(args)
    line['breakout'] = breakout_section(args)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
