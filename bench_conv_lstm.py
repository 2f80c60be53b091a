#!/usr/bin/env python
"""bench_conv_lstm.py -- the reference's Atari LSTM policy, RecurrentPolicy(LSTMWrapper(Convolutional(env), 512, 512)),
trained on the 'cudnn_conv' plan (conv1 on the bptt segments where the rollout left them, the fused PPO loss, train()
captured) against today's plan for it, which fused_loss=False reproduces ('cudnn': b_obs gathered, the reference
autograd loss, eager).  cuda_graph=True, bptt 16, 4 minibatches x 4 epochs (bench.ppo_config).

    python bench_conv_lstm.py [--reps K] [--skip-c4] [--skip-profile]

Prints one JSON line with the card's name and power limit and
  * `ppo`: evaluate() + train() and train() alone, agent-steps/s, on pong and breakout_pixels at 1 024 x 128, the two
    trainers alternated in one process (CUDA events around each call, median);
  * `c4`: 4 096 x 128 on pong and breakout_pixels, each plan alone in a fresh process, with peak memory, both graph
    states and this project's kernel launches per train() (from Python, and inside the captured graph);
  * `profile`: per-op CUDA time (torch.profiler, in a process of its own) of one C4 minibatch's (8 192 segments x 16
    steps = 131 072 rows) forward + loss + backward on each plan.
Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

import torch

from bench import gpu_info, ppo_config
from bench_pong import summary, timed

PLANS = ('cudnn_conv', 'today')


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=6, help='timed evaluate() + train() calls per trainer')
    ap.add_argument('--skip-c4', action='store_true')
    ap.add_argument('--skip-profile', action='store_true')
    ap.add_argument('--c4', nargs=2, metavar=('ENV', 'PLAN'), help='run C4 of ENV on PLAN (cudnn_conv / today) alone')
    ap.add_argument('--profile-only', action='store_true')
    return ap.parse_args()


def make_trainer(env, n, h, plan):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    net = models.LSTMWrapper(vec.driver_env, models.Convolutional(vec.driver_env), input_size=512, hidden_size=512)
    policy = cleanrl.RecurrentPolicy(net, seed=1).cuda()
    cfg = ppo_config(n, h, 'cuda', seed=1, cuda_graph=True, env=env)
    cfg.fused_loss = plan == 'cudnn_conv'
    return cp.create(cfg, vec, policy)


def states(d):
    return dict(train_graph_state=d.train_graph_state, rollout_graph_state=d.graph_state,
                minibatch_path=d.train_minibatch_path, msg=d.msg or None)


def launches_per_train(cp, d):
    from pufferlib_b200 import _native
    lib = _native.lib()
    cp.evaluate(d)
    torch.cuda.synchronize()
    l0 = lib.pb_launch_count()
    cp.train(d)
    torch.cuda.synchronize()
    from_python = int(lib.pb_launch_count() - l0)
    return dict(from_python=from_python, in_graph=int(d.train_graph_launches) if d.train_graph_state == 2 else 0)


def alternated(args, env):
    from pufferlib_b200 import clean_pufferl as cp
    n, h = 1024, 128
    runs = {p: make_trainer(env, n, h, p) for p in PLANS}
    for d in runs.values():
        for _ in range(3):
            cp.evaluate(d)
            cp.train(d)
    both, train = {k: [] for k in runs}, {k: [] for k in runs}
    for _ in range(args.reps):
        for k, d in runs.items():
            timed(cp, d, both[k], train[k])
    a = dict(num_envs=n, horizon=h, statistic='median', **{
        k: dict(summary(n * h, both[k], train[k]), **states(d)) for k, d in runs.items()})
    a['speedup_evaluate_train'] = a['cudnn_conv']['agent_steps_per_s'] / a['today']['agent_steps_per_s']
    a['speedup_train'] = a['cudnn_conv']['train_agent_steps_per_s'] / a['today']['train_agent_steps_per_s']
    for d in runs.values():
        cp.close(d)
    del runs
    torch.cuda.empty_cache()
    return a


def c4_run(args, env, plan):
    from pufferlib_b200 import clean_pufferl as cp
    n, h = 4096, 128
    torch.cuda.reset_peak_memory_stats()
    d = make_trainer(env, n, h, plan)
    for _ in range(2):
        cp.evaluate(d)
        cp.train(d)
    launches = launches_per_train(cp, d)
    b_, t_ = [], []
    for _ in range(max(2, args.reps // 2)):
        timed(cp, d, b_, t_)
    return dict(summary(n * h, b_, t_), **states(d), launches_per_train=launches,
                b_obs_allocated=d.experience._b_obs is not None,
                max_memory_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def profile_section():
    """One C4 minibatch's forward + loss + backward, per-op CUDA time, each plan after a warm-up call: 'cudnn_conv' on the
    segment view of a 4 096 x 128 rollout buffer with fused_ppo_loss, 'today' on the gathered copy (b_obs[mb]) through
    RecurrentPolicy with the reference loss."""
    import pufferlib_b200
    from torch.profiler import ProfilerActivity, profile
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.frameworks import cleanrl
    from bench_nature_trunk import fake_env
    n, h, bptt, nm, mb = 4096, 128, 16, 4, 1
    g_ = h // bptt // nm
    obs = torch.randint(0, 256, (h * n, 4, 84, 84), dtype=torch.uint8, device='cuda')
    view = obs.view(g_, nm, bptt, n, 4, 84, 84)[:, mb].permute(2, 0, 1, 3, 4, 5)
    rows, segs = n * g_ * bptt, n * g_
    # the shapes train() hands over: actions and logprobs [segments, bptt] (b_actions[mb]), the rest [rows]
    atn, old_lp = torch.randint(0, 6, (segs, bptt), device='cuda'), -torch.rand(segs, bptt, device='cuda') - 1.0
    adv, ret, old_v = (torch.randn(rows, device='cuda') for _ in range(3))
    cfg = pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    out = dict(rows=rows, segments=segs, steps=bptt)
    for plan in PLANS:
        torch.manual_seed(0)
        net = models.LSTMWrapper(fake_env(), models.Convolutional(fake_env()), input_size=512, hidden_size=512).cuda()
        pol = cleanrl.RecurrentPolicy(net)
        x = view if plan == 'cudnn_conv' else view.contiguous().view(segs, bptt, 4, 84, 84)

        def step():
            if plan == 'cudnn_conv':
                logits, value, _ = net.forward_segments(x, None)
                loss, _ = cp.fused_ppo_loss(logits, value, atn, old_lp, adv, ret, old_v, cfg)
            else:
                _, lp, ent, value, _ = pol(x, state=None, action=atn)
                loss, _ = cp._ppo_loss(lp, ent, value, old_lp, adv, ret, old_v, cfg)
            loss.backward()
        step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        ops = []
        for ev in prof.key_averages():
            us = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0)
            if us > 0 and ev.key and not ev.key.startswith('aten::') and 'Memcpy' not in ev.key:
                ops.append((ev.key[:90], us / 1e3, ev.count))
        ops.sort(key=lambda r: -r[1])
        out[plan] = dict(total_ms=sum(r[1] for r in ops), ops=[dict(name=k, ms=t_, calls=c) for k, t_, c in ops[:16]],
                         max_memory_allocated_gib=torch.cuda.max_memory_allocated() / 2 ** 30)
        del net, pol, x
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    return out


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
    if args.profile_only:
        torch.cuda.set_device(0)
        print(json.dumps(profile_section()))
        return
    line = {}
    if not args.skip_c4:       # before this process touches the device
        c4 = {}
        for env in ('pong', 'breakout_pixels'):
            c4[env] = {p: subprocess_json(['--c4', env, p, '--reps', str(args.reps)]) for p in PLANS}
            r = c4[env]
            if all('agent_steps_per_s' in r[p] for p in PLANS):
                r['speedup_evaluate_train'] = r['cudnn_conv']['agent_steps_per_s'] / r['today']['agent_steps_per_s']
                r['speedup_train'] = r['cudnn_conv']['train_agent_steps_per_s'] / r['today']['train_agent_steps_per_s']
        line['c4'] = c4
    if not args.skip_profile:
        line['profile'] = subprocess_json(['--profile-only'])
    torch.cuda.set_device(0)
    line['gpu'] = gpu_info(0)
    line['method'] = 'CUDA events around evaluate()/train() calls, median; torch.profiler for the per-op split'
    line['ppo'] = {env: alternated(args, env) for env in ('pong', 'breakout_pixels')}
    print(json.dumps(line))


if __name__ == '__main__':
    main()
