#!/usr/bin/env python
"""bench_lstm_ranks.py -- the recurrent update as rank 0 of 2 on ONE device, the other rank's half of the exchange staged in
local memory (tests/util_peer.py).

    python bench_lstm_ranks.py [--num-envs N] [--horizon H] [--train-reps R] [--kernel-reps K]

Prints one JSON line with
  * `kernel`: pb_peer_allreduce_mean (16 CTAs) per call at the flat gradient sizes of LSTMWrapper(Default): 149 253 floats
    (H = 128, F = 128, 4 actions) and 560 645 (H = 256).  The peer buffers are on the same device, so this is the kernel's
    LOCAL-memory time, not an NVLink time: K back-to-back calls between two CUDA events, flags staged ahead so no call
    waits, best of 3.
  * `train`: train() of RecurrentPolicy(LSTMWrapper(Default), fused_sample=True, fused_update=True) on breakout (bench_lstm.py's
    shape: 16 384 envs x 128 steps, 4 minibatches, 4 epochs), captured in one CUDA graph vs eager, as rank 0 of 2 with the
    peer exchange: two trainers built the same way in one process and alternated, CUDA events around each call, median.
    Both run the same kernels; the exchange costs one local-memory kernel per minibatch here, so the time on two real
    GPUs (NVLink) is not measured by this script.
The card's name and power limit go with the numbers.  Writes nothing to the tree.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

from bench import gpu_info, ppo_config

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'tests'))
import util_peer as up  # noqa: E402

WORLD, RANK = 2, 0


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-envs', type=int, default=16384)
    ap.add_argument('--horizon', type=int, default=128)
    ap.add_argument('--train-reps', type=int, default=10, help='timed train() calls per trainer (captured, eager)')
    ap.add_argument('--kernel-reps', type=int, default=200, help='kernel calls per timed window')
    return ap.parse_args()


def stage_ahead(peers, n, steps):
    """Zero peer gradients in both slots and every peer flag at the last epoch the next `steps` exchanges reach."""
    zero = torch.zeros(WORLD, n, device='cuda')
    last = peers.epoch + steps
    for parity in (0, 1):
        peers._stage(parity, zero, n, last)
    torch.cuda.synchronize()


def kernel_time(n, reps):
    from pufferlib_b200 import _native
    lib = _native.lib()
    peers = up.StagedPeers(WORLD, RANK, (n + 3) // 4 * 4 + 4, torch.device('cuda'), sliced=True)
    flat = torch.randn(n, device='cuda')
    best = float('inf')
    for _ in range(4):                     # the first window warms up
        stage_ahead(peers, n, reps)
        s = torch.cuda.current_stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            _native.check(lib.pb_peer_allreduce_mean(C.byref(peers.struct), _native.ptr(flat), n, None, None,
                                                     _native.stream_ptr(s)))
        e1.record()
        torch.cuda.synchronize()
        peers.epoch += reps
        peers.check_epoch()
        best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
    return best


class Ranks:
    """torch.distributed as rank 0 of 2 without a process group; distributed.PeerComm -> staged peers."""

    def __init__(self, exchanges_per_train):
        import torch.distributed as dist
        import pufferlib_b200.distributed as pdist
        dist.is_initialized = lambda: True
        dist.get_world_size = lambda group=None: WORLD
        dist.get_rank = lambda group=None: RANK
        dist.all_reduce = lambda tensor, op=None, group=None, async_op=False: None
        self.per_train = exchanges_per_train
        self.made = []

        def staged(capacity):
            peers = up.StagedPeers(WORLD, RANK, capacity, torch.device('cuda'), sliced=True)
            peers.close = lambda: None
            peers.n = capacity - 4
            stage_ahead(peers, peers.n, self.per_train)
            self.made.append(peers)
            return peers
        pdist.PeerComm = staged


def make_trainer(args, captured):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    n, h = args.num_envs, args.horizon
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
    policy = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1, fused_update=True).cuda()
    cfg = ppo_config(n, h, 'cuda', seed=1, cuda_graph=True)
    cfg.cuda_graph_train = captured
    return cp.create(cfg, vec, policy)


def main(args):
    from pufferlib_b200 import _native, clean_pufferl as cp
    torch.cuda.set_device(0)
    kernel = {str(n): round(kernel_time(n, args.kernel_reps), 2) for n in (149253, 560645)}
    cfg = ppo_config(args.num_envs, args.horizon, 'cuda')
    per_train = cfg.update_epochs * (cfg.batch_size // cfg.minibatch_size)
    ranks = Ranks(per_train)
    runs = {'captured': make_trainer(args, True), 'eager': make_trainer(args, False)}
    peers = {}
    times = {k: [] for k in runs}
    for i in range(args.train_reps + 2):     # call 0 eager on both, call 1 captures; two warm-ups
        for k, d in runs.items():
            if k in peers:
                stage_ahead(peers[k], peers[k].n, per_train)
            cp.evaluate(d)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            cp.train(d)
            e1.record()
            torch.cuda.synchronize()
            if k not in peers:
                peers[k] = d.grad_bucket.peer
            peers[k].epoch += per_train
            peers[k].check_epoch()
            if i >= 2:
                times[k].append(e0.elapsed_time(e1))
    plans = {k: tuple(getattr(cp.update_plan(d), a) for a in ('engine', 'form', 'capture')) for k, d in runs.items()}
    assert plans['captured'] == ('bptt', 'segments', 'whole') and runs['captured'].train_graph_state == 2, plans
    assert len(ranks.made) == 2 and all(d.grad_bucket.peer is not None for d in runs.values())
    launches = {}
    for k, d in runs.items():
        stage_ahead(peers[k], peers[k].n, per_train)
        cp.evaluate(d)
        torch.cuda.synchronize()
        l0 = _native.lib().pb_launch_count()
        cp.train(d)
        torch.cuda.synchronize()
        launches[k] = int(_native.lib().pb_launch_count() - l0)
        peers[k].epoch += per_train
        peers[k].check_epoch()
    med = {k: float(np.median(v)) for k, v in times.items()}
    line = {
        'metric': 'train_ms_rank0_of_2', 'unit': 'ms', 'gpu': gpu_info(0),
        'config': {'workload': f'breakout num_envs={args.num_envs} horizon={args.horizon} RecurrentPolicy(LSTMWrapper(Default)) '
                               'hidden=128 fused_update=True, rank 0 of 2 with staged peers', 'minibatches': 4, 'epochs': 4,
                   'exchanges_per_train': per_train, 'train_reps': args.train_reps},
        'kernel_us_local_memory': kernel,
        'train_ms': {k: round(v, 3) for k, v in med.items()},
        'train_ms_all': {k: [round(x, 3) for x in v] for k, v in times.items()},
        'captured_over_eager': round(med['captured'] / med['eager'], 4),
        'project_launches_per_train': launches,
        'plans': plans,
    }
    for d in runs.values():
        cp.close(d)
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main(parse_args())
