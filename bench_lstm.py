#!/usr/bin/env python
"""bench_lstm.py -- the recurrent policy on the device path: RecurrentPolicy(LSTMWrapper(Default), fused_sample=True).

    python bench_lstm.py [--env breakout|squared] [--num-envs N] [--horizon H] [--steps K] [--warmup W]

Prints one JSON line with
  * agent-steps/s of the PPO loop (CUDA-graphed rollout, recurrent update on cuDNN autograd), the same step definition
    as bench.py;
  * `policy_step`: the rollout-time policy step, fused (pb_policy_lstm_sample: one kernel) vs unfused
    (fused_sample=False), measured in the same process on the rollout's own observation rows;
  * `roofline_kernels.policy_lstm_step`: algorithmic HBM bytes 4F + 2048 + 16 per row over the fused step time, against
    the H100 SXM data-sheet 3.35 TB/s; the packed weights each CTA streams from L2 are reported separately.
Shared pieces (PPO config, timed steps, card name and power limit) come from bench.py.  Writes nothing to the tree.
"""
import argparse
import json

import numpy as np
import torch

from bench import METRIC, UNIT, gpu_info, ppo_config, timed_steps


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--env', default='breakout', choices=['breakout', 'squared'])
    ap.add_argument('--num-envs', type=int, default=16384)
    ap.add_argument('--horizon', type=int, default=128)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--minibatches', type=int, default=4, help='batch_size / minibatch_size (reference ratio: 4)')
    ap.add_argument('--epochs', type=int, default=4)
    ap.add_argument('--no-graph', action='store_true')
    ap.add_argument('--reps', type=int, default=256, help='policy steps per timed CUDA graph')
    return ap.parse_args()


def policy_step_times(data, reps=256):
    """Device time of one rollout-time policy step of the recurrent policy, fused (pb_policy_lstm_sample: one kernel) and
    unfused (fused_sample=False: encoder GEMM, cuDNN LSTM, head GEMM, sample_logits, the h / c copies back into the
    rollout state and the row store, as clean_pufferl._rollout_loop runs it), in the same process on the rollout's own
    observation rows.  `reps` steps are captured into a CUDA graph and replayed between two CUDA events (warmed up, best
    of 3); if the unfused chain cannot be captured it is timed eagerly, launch overhead included, and `method` says so."""
    from pufferlib_b200 import _native
    policy, exp = data.policy, data.experience
    n = exp.num_envs
    h = exp.batch_size // n
    obs_rows = [exp.obs[t * n:(t + 1) * n] for t in range(h)]
    hs, cs = exp.lstm_h.clone(), exp.lstm_c.clone()       # scratch state: the rollout's own state is left as it is
    outs = (torch.empty(n, device='cuda'), torch.empty(n, device='cuda'), torch.empty(n, dtype=torch.int64, device='cuda'))
    lib = _native.lib()

    def step(fused, i):
        x = obs_rows[i % h]
        if fused:
            policy(x, (hs, cs), out=outs)
        else:
            a, lp, _, v, (h2, c2) = policy(x, (hs, cs))
            hs.copy_(h2)
            cs.copy_(c2)
            v = v.reshape(-1)
            _native.check(lib.pb_rollout_store(_native.ptr(v), _native.ptr(lp), _native.ptr(a), _native.ptr(outs[0]),
                                               _native.ptr(outs[1]), _native.ptr(outs[2]), n, _native.stream_ptr()))

    def best_of_3(run):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        best = float('inf')
        for _ in range(3):
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1))
        return best / reps * 1e-3

    res = {}
    fused0 = policy.fused_sample
    try:
        for fused in (True, False):
            policy.fused_sample = fused
            with torch.no_grad():
                for i in range(8):
                    step(fused, i)                                      # warm-up: module loads, library algorithm picks
                torch.cuda.synchronize()
                eager = best_of_3(lambda: [step(fused, i) for i in range(reps)])
                try:
                    policy.policy.invalidate_cache()                    # packed operands are rebuilt inside the capture
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        for i in range(reps):
                            step(fused, i)
                    g.replay()
                    torch.cuda.synchronize()
                    graphed, method = best_of_3(g.replay), 'cuda graph of %d steps, best of 3 replays' % reps
                    del g
                except Exception as e:                                  # reported in `method`, not hidden
                    graphed, method = None, f'eager only (capture failed: {type(e).__name__})'
                policy.policy.invalidate_cache()
            res['fused' if fused else 'unfused'] = {'seconds': graphed if graphed is not None else eager,
                                                    'eager_seconds': eager, 'method': method}
    finally:
        policy.fused_sample = fused0
    return res


def main(args):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    torch.cuda.set_device(0)
    n, h = args.num_envs, args.horizon
    vec = pvec.make(ocean.env_creator(args.env), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env, hidden_size=128), input_size=128,
                             hidden_size=128)
    policy = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1).cuda()
    cfg = ppo_config(n, h, 'cuda', seed=1, cuda_graph=not args.no_graph, minibatches=args.minibatches,
                     epochs=args.epochs, env=args.env)
    data = cp.create(cfg, vec, policy)
    for _ in range(max(args.warmup, 2)):
        cp.evaluate(data)
        cp.train(data)
    ms = timed_steps(data, cp, args.steps, 1)
    prof = {k: round(v, 4) for k, v in dict(data.profile).items() if k.endswith('_time')}
    times = policy_step_times(data, args.reps)
    # algorithmic HBM bytes of one fused step: x (4F), h and c read and written (4 x 512), value + logprob + action (16)
    feats = int(np.prod(vec.single_observation_space.shape))
    step_bytes = n * (4 * feats + 2048 + 16)
    peak_gbs = 3350.0
    bound_s = step_bytes / (peak_gbs * 1e9)
    t_f, t_u = times['fused']['seconds'], times['unfused']['seconds']
    ctas = -(-n // 128)
    # packed operands one CTA reads from L2 (W_enc, gate weights, biases, 16-row head matrix): not HBM traffic per step
    weight_bytes = 4 * (128 * 136 + 16 * 32 * 264 + 128 + 512 + 16 * 128 + 16)
    line = {
        'metric': METRIC, 'value': n * h * args.steps / (ms * 1e-3), 'unit': UNIT, 'n_gpus': 1, 'steps': args.steps,
        'warmup': max(args.warmup, 2), 'ms_per_step': ms / args.steps, 'higher_is_better': True,
        'config': {'workload': f'{args.env} num_envs={n} horizon={h} RecurrentPolicy(LSTMWrapper(Default)) hidden=128 '
                               'fused_sample=True', 'global_batch': n * h, 'minibatch_size': n * h // args.minibatches,
                   'update_epochs': args.epochs, 'bptt_horizon': 16, 'cuda_graph_rollout': not args.no_graph,
                   'update': 'cuDNN LSTM autograd'},
        'policy_step': {
            'fused_us': round(t_f * 1e6, 2), 'unfused_us': round(t_u * 1e6, 2), 'speedup': round(t_u / t_f, 2),
            'fused_eager_us': round(times['fused']['eager_seconds'] * 1e6, 2),
            'unfused_eager_us': round(times['unfused']['eager_seconds'] * 1e6, 2),
            'method': {k: v['method'] for k, v in times.items()}},
        'roofline_kernels': {'policy_lstm_step': {
            'kernel': 'k_policy_lstm_sample', 'algorithmic_bytes_per_launch': step_bytes,
            'bytes_per_row': 4 * feats + 2048 + 16, 'hbm_bound_us': round(bound_s * 1e6, 2),
            'peak': peak_gbs, 'peak_source': 'H100 SXM5 HBM3 data sheet (3.35 TB/s), not measured',
            'avg_launch_us': round(t_f * 1e6, 2), 'achieved': round(step_bytes / t_f / 1e9, 1),
            'frac': round(bound_s / t_f, 4), 'launches_per_step': h,
            'l2_weight_bytes_per_cta': weight_bytes, 'l2_weight_bytes_per_launch': weight_bytes * ctas}},
        'gpu': gpu_info(0), 'profile_s': prof, 'env_stats': {k: float(v) for k, v in data.stats.items()},
    }
    print(json.dumps(line))
    cp.close(data)


if __name__ == '__main__':
    main(parse_args())
