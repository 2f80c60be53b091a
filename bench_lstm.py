#!/usr/bin/env python
"""bench_lstm.py -- the recurrent policy on the device path: RecurrentPolicy(LSTMWrapper(Default), fused_sample=True).

    python bench_lstm.py [--env breakout|squared] [--num-envs N] [--horizon H] [--steps K] [--warmup W] [--fused-update]

Prints one JSON line with
  * agent-steps/s of the PPO loop (CUDA-graphed rollout; recurrent update on cuDNN autograd, or with --fused-update on
    the BPTT kernels pb_lstm_bptt_forward / _backward + pb_ppo_loss), the same step definition as bench.py;
  * `policy_step`: the rollout-time policy step, fused (pb_policy_lstm_sample: one kernel) vs unfused
    (fused_sample=False), measured in the same process on the rollout's own observation rows;
  * `roofline_kernels.policy_lstm_step`: algorithmic HBM bytes 4F + 2048 + 16 per row over the fused step time, against
    the H100 SXM data-sheet 3.35 TB/s; the packed weights each CTA streams from L2 are reported separately;
  * `update`: forward + loss + backward of one training minibatch ([B segments, T = 16 steps] of the rollout), fused
    (forward_packed_seq on the minibatch form train() used: the segment view of the rollout buffer, or the gathered
    copy) + fused_ppo_loss_packed vs cuDNN (the LSTMWrapper forward on the gathered segments + the autograd loss, as
    train() runs it), in the same process on the same minibatch, from CUDA events; with the algorithmic bytes and TF32
    FLOPs per row of the fused path and the share of each data-sheet bound;
  * `train` (with --fused-update and graphs): train() alone, captured in one CUDA graph vs eager, on two trainers built
    the same way in one process and alternated, CUDA events around each call, median; the project's kernel launches per
    train() (pb_launch_count), the peak memory each kind of call allocates beyond what was allocated before it, and the
    observation bytes the segment view no longer gathers.
Shared pieces (PPO config, timed steps, card name and power limit) come from bench.py.  Writes nothing to the tree.
"""
import argparse
import json

import numpy as np
import torch

from bench import METRIC, UNIT, gpu_info, ppo_config, timed_steps


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--env', default='breakout', choices=['breakout', 'squared', 'memory'])
    ap.add_argument('--num-envs', type=int, default=16384)
    ap.add_argument('--horizon', type=int, default=128)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--minibatches', type=int, default=4, help='batch_size / minibatch_size (reference ratio: 4)')
    ap.add_argument('--epochs', type=int, default=4)
    ap.add_argument('--no-graph', action='store_true')
    ap.add_argument('--reps', type=int, default=256, help='policy steps per timed CUDA graph')
    ap.add_argument('--fused-update', action='store_true', help='train() on the fused BPTT kernels')
    ap.add_argument('--update-reps', type=int, default=10, help='timed minibatch updates per path')
    ap.add_argument('--train-reps', type=int, default=10, help='timed train() calls per trainer (captured, eager)')
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


def update_cost_per_row(feats, n_out, steps):
    """Algorithmic HBM bytes and TF32 tensor-core FLOPs per minibatch row of the fused update (forward kernel, loss
    kernel, backward kernel, weight-gradient GEMMs and column sums), from the shapes.  n_out = R head columns."""
    H, G = 128, 512
    state = 4 * 4 * H / steps                                   # h0, c0 read and h_T, c_T written, once per segment
    nbytes = {
        'forward': 4 * feats + 4 * 1024 + 4 * n_out + state,     # x; saved row written; out written
        'loss': 4 * n_out + 28 + 4 * n_out,                     # out + 7 per-row scalars read; dOut written
        'backward': 4 * n_out + 4 * (H + 4 * H + H) + 4 * G + 4 * H,   # dOut, e, activations, c read; dz, dPre written
        'weight_grads': 2 * 4 * G + 4 * 2 * H + 2 * 4 * H + 4 * feats + 2 * 4 * n_out + 4 * H,
        # dz (GEMM + column sum), [e | h_prev], dPre (GEMM + sum), x, dOut (GEMM + sum), h
    }
    flops = {
        'forward': 2 * (feats * H + 2 * H * G + H * n_out),      # encoder, gates, heads
        'backward': 2 * (G * 2 * H),                              # dz [W_ih | W_hh]
        'weight_grads': 2 * (G * 2 * H + H * feats + n_out * H),  # dW_ih | dW_hh, dW_enc, dW_cat
    }
    return nbytes, flops


def update_times(data, reps=10):
    """Device time of forward + loss + backward of one training minibatch (minibatch 0 of the last train(), initial
    state None), fused (forward_packed_seq on the minibatch form the last train() read + fused_ppo_loss_packed +
    backward) and cuDNN (the RecurrentPolicy forward over the gathered segments + the autograd loss of train() +
    backward), alternating, each bracketed by CUDA events; median of `reps` after 2 warm-ups.  The optimizer step is not
    included.  -> (times, (segments, bptt), minibatch form)."""
    from pufferlib_b200 import clean_pufferl as cp
    policy, exp, cfg = data.policy, data.experience, data.config
    form = data.train_minibatch_path
    if form == 'segments':       # [E, G, T, *obs] view of the rollout buffer; the cuDNN forward gets a gathered copy
        seg = exp.segment_obs(0)
        obs, obs_g = seg, seg.reshape(-1, *seg.shape[2:])
    else:
        obs = obs_g = exp.b_obs[0]
    atn, lp = exp.b_actions[0], exp.b_logprobs[0]
    val, ret, adv = exp.b_values[0], exp.b_returns[0], exp.b_advantages[0]
    model = policy.policy

    def fused():
        out, n_act, _ = model.forward_packed_seq(obs, None)
        loss, _ = cp.fused_ppo_loss_packed(out, n_act, atn, lp, adv, ret, val, cfg)
        loss.backward()

    def cudnn():
        _, newlogprob, entropy, newvalue, _ = policy(obs_g, state=None, action=atn)
        ratio = (newlogprob - lp.reshape(-1)).exp()
        a = adv.reshape(-1)
        pg = torch.max(-a * ratio, -a * torch.clamp(ratio, 1 - cfg.clip_coef, 1 + cfg.clip_coef)).mean()
        v = newvalue.view(-1)
        r = ret.reshape(-1)
        vc = val.reshape(-1) + torch.clamp(v - val.reshape(-1), -cfg.vf_clip_coef, cfg.vf_clip_coef)
        v_loss = 0.5 * torch.max((v - r) ** 2, (vc - r) ** 2).mean()
        (pg - cfg.ent_coef * entropy.mean() + v_loss * cfg.vf_coef).backward()

    runs = {'fused': fused, 'cudnn': cudnn}
    times = {k: [] for k in runs}
    for i in range(reps + 2):
        for k, run in runs.items():
            policy.zero_grad(set_to_none=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            if i >= 2:
                times[k].append(e0.elapsed_time(e1) * 1e-3)
    policy.zero_grad(set_to_none=True)
    return {k: float(np.median(v)) for k, v in times.items()}, tuple(obs_g.shape[:2]), form


def make_trainer(args, train_graph):
    """Vecenv, RecurrentPolicy(LSTMWrapper(Default)) and trainer, the same for every call but for `train_graph`
    (config.cuda_graph_train); the rollout is captured unless --no-graph."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    n, h = args.num_envs, args.horizon
    vec = pvec.make(ocean.env_creator(args.env), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env, hidden_size=128), input_size=128,
                             hidden_size=128)
    policy = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1, fused_update=args.fused_update).cuda()
    cfg = ppo_config(n, h, 'cuda', seed=1, cuda_graph=not args.no_graph, minibatches=args.minibatches,
                     epochs=args.epochs, env=args.env)
    cfg.cuda_graph_train = train_graph
    return cp.create(cfg, vec, policy)


def train_peak(cp, data):
    """One train(); -> (bytes allocated at its peak beyond what was allocated before it, pb_launch_count delta)."""
    from pufferlib_b200 import _native
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base, l0 = torch.cuda.memory_allocated(), _native.lib().pb_launch_count()
    cp.train(data)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, _native.lib().pb_launch_count() - l0


def train_times(args, graphed):
    """train() alone, captured (`graphed`, already warmed up: eager call, then capture + first replay) vs eager (a
    second trainer built the same way, config.cuda_graph_train=False), alternating; each call after its own rollout,
    bracketed by CUDA events (train() ends in its one device-to-host read, so the events span the whole call, host
    launch gaps included); median of --train-reps after 2 warm-ups per trainer."""
    from pufferlib_b200 import clean_pufferl as cp
    eager = make_trainer(args, train_graph=False)
    runs = {'captured': graphed, 'eager': eager}
    times = {k: [] for k in runs}
    peaks, launches = {}, {}
    for i in range(args.train_reps + 2):
        for k, d in runs.items():
            cp.evaluate(d)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            cp.train(d)
            e1.record()
            torch.cuda.synchronize()
            if i >= 2:
                times[k].append(e0.elapsed_time(e1) * 1e-3)
    for k, d in runs.items():            # one more call each, untimed: memory and launches
        cp.evaluate(d)
        peaks[k], launches[k] = train_peak(cp, d)
    state, paths = eager.train_graph_state, (graphed.train_recurrent_path, eager.train_recurrent_path)
    cp.close(eager)
    return {k: float(np.median(v)) for k, v in times.items()}, peaks, launches, state, paths


def main(args):
    from pufferlib_b200 import clean_pufferl as cp
    torch.cuda.set_device(0)
    n, h = args.num_envs, args.horizon
    data = make_trainer(args, train_graph=not args.no_graph)
    vec, policy = data.vecenv, data.policy
    warm_peaks = []           # per warm-up train(): the first is eager; with a captured update the second captures
    for _ in range(max(args.warmup, 2)):
        cp.evaluate(data)
        warm_peaks.append(train_peak(cp, data)[0])
    ms = timed_steps(data, cp, args.steps, 1)
    prof = {k: round(v, 4) for k, v in dict(data.profile).items() if k.endswith('_time')}
    recurrent_path, minibatch_path = data.train_recurrent_path, data.train_minibatch_path
    times = policy_step_times(data, args.reps)
    upd, (seg, bptt), form = update_times(data, args.update_reps)
    n_act = vec.single_action_space.n
    n_out = -(-(n_act + 1) // 8) * 8
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
                   'update': 'fused BPTT kernels' if args.fused_update else 'cuDNN LSTM autograd',
                   'train_recurrent_path': recurrent_path, 'train_minibatch_path': minibatch_path,
                   'train_graph_state': data.train_graph_state},
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
        'update': dict(update_section(upd, seg, bptt, feats, n_out), fused_minibatch_form=form),
        'train': train_section(args, data, warm_peaks, feats),
        'gpu': gpu_info(0), 'profile_s': prof, 'env_stats': {k: float(v) for k, v in data.stats.items()},
    }
    if args.env == 'memory':
        line['memory_env_step'] = memory_env_step_times(n)
    print(json.dumps(line))
    cp.close(data)


def memory_env_step_times(n, cycles=20):
    """The memory env step alone (no policy), CUDA events around each send: a step-send vs a reset-send.  At the
    default mem_length=2, mem_delay=2 every episode is 5 steps and all envs reset together, so every 6th send is a
    reset-send; it also regenerates N * 6 outputs of the shared MT19937 stream in one CTA (k_mem_prepare)."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200.environments import ocean
    vec = pvec.make(ocean.env_creator('memory'), num_envs=n, backend=pvec.B200)
    actions = torch.zeros(n, dtype=torch.int64, device='cuda')
    vec.async_reset(1)
    vec.recv()
    times = {'step': [], 'reset': []}
    for k in range(6 * cycles):
        reset = k % 6 == 5
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        vec.send(actions)
        b.record()
        vec.recv()
        b.synchronize()
        times['reset' if reset else 'step'].append(a.elapsed_time(b) * 1e3)
    vec.close()
    med = {k: float(np.median(v)) for k, v in times.items()}
    return {'step_send_us': round(med['step'], 2), 'reset_send_us': round(med['reset'], 2),
            'mt_outputs_per_reset_send': n * 6, 'mt_twists_per_reset_send': round(n * 6 / 624, 1),
            'method': f'median of {len(times["step"])} step-sends and {len(times["reset"])} reset-sends, CUDA events '
                      'around send() (env kernels + host launch), after warm-up by the PPO loop in the same process'}


def train_section(args, data, warm_peaks, feats):
    n, h = args.num_envs, args.horizon
    if data.train_graph_state != 2:
        return {'skipped': f'the update of this run is not captured (train_graph_state {data.train_graph_state}, path '
                           f'{data.train_recurrent_path}; captured updates need --fused-update and graphs)'}
    t, peaks, launches, eager_state, paths = train_times(args, data)
    gather_bytes = 2 * h * n * 4 * feats           # pb_minibatch_gather: every observation row read once, written once
    return {
        'captured_ms': round(t['captured'] * 1e3, 3), 'eager_ms': round(t['eager'] * 1e3, 3),
        'eager_over_captured': round(t['eager'] / t['captured'], 3),
        'method': 'train() alone, two trainers built the same way, alternated; CUDA events around each call, median of '
                  f'{args.train_reps}',
        'recurrent_path': {'captured': paths[0], 'eager': paths[1]}, 'eager_train_graph_state': eager_state,
        'launches_per_train': {'captured': {'graph_launches': 1, 'project_kernels_in_graph': data.train_graph_launches,
                                            'project_kernels_launched_from_python': launches['captured']},
                               'eager': {'project_kernels_launched_from_python': launches['eager']},
                               'note': 'pb_launch_count counts this project\'s kernels only, not torch / cuBLAS ones'},
        'peak_bytes_beyond_allocated': {'eager_first_call': warm_peaks[0], 'capture_call': warm_peaks[1],
                                        'replay': peaks['captured'], 'eager': peaks['eager']},
        'obs_gather_bytes_saved_per_train': gather_bytes, 'b_obs_bytes_not_allocated': h * n * 4 * feats,
    }


def update_section(upd, seg, bptt, feats, n_out):
    rows = seg * bptt
    nbytes, flops = update_cost_per_row(feats, n_out, bptt)
    b_row, f_row = sum(nbytes.values()), sum(flops.values())
    peak_gbs, peak_tflops = 3350.0, 495.0
    t_bytes, t_flops = rows * b_row / (peak_gbs * 1e9), rows * f_row / (peak_tflops * 1e12)
    t_f, t_c = upd['fused'], upd['cudnn']
    return {
        'minibatch': {'segments': seg, 'bptt': bptt, 'rows': rows},
        'fused_ms': round(t_f * 1e3, 3), 'cudnn_ms': round(t_c * 1e3, 3), 'speedup': round(t_c / t_f, 2),
        'method': 'forward + loss + backward per minibatch (no optimizer step), CUDA events, median',
        'bytes_per_row': nbytes, 'tf32_flops_per_row': flops,
        'hbm_bound_ms': round(t_bytes * 1e3, 3), 'tf32_bound_ms': round(t_flops * 1e3, 3),
        'share_of_hbm_bound': round(t_bytes / t_f, 4), 'share_of_tf32_bound': round(t_flops / t_f, 4),
        'bound_by': 'hbm' if t_bytes >= t_flops else 'tf32',
        'peak_source': 'H100 SXM5 data sheet: 3.35 TB/s HBM3, 495 TFLOP/s dense TF32 (700 W); not measured',
    }


if __name__ == '__main__':
    main(parse_args())
