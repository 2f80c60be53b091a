#!/usr/bin/env python
"""bench_target_kl.py -- train() with target_kl set, on bench.py's workload (breakout, 16 384 envs x 128 steps, 4
minibatches x 4 epochs).

    python bench_target_kl.py [--num-envs N] [--horizon H] [--reps K]

Two trainers built the same way in one process and alternated: `autograd_eager` (manual_update=False and
cuda_graph_train=False: autograd, clip_grad_norm_ and torch.optim.Adam, eager, the host reading the stop flag after every
epoch -- what a trainer with target_kl ran before the stop moved to the device) and `captured` (the default plan: the
hand-written update, captured in one graph, the later epochs inside IF nodes).  Each trainer collects one rollout and
keeps it; every timed train() starts from the same parameters and Adam state (restored outside the timed window), so
every call makes the same decisions.  Two settings of target_kl: `never` (1e9: all 4 epochs, the work of target_kl=None)
and `after_epoch_1` (between the last minibatch's approx_kl of epoch 0 and of epoch 1, read from one eager probe call per
trainer).  Prints one JSON line: per setting and trainer the median train() time (CUDA events, --reps calls) and its min /
max, the epochs run, and the speedup.  The card's name and power limit go with the numbers.  Writes nothing to the tree."""
import argparse
import json

import numpy as np
import torch

from bench import gpu_info, ppo_config


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-envs', type=int, default=16384)
    ap.add_argument('--horizon', type=int, default=128)
    ap.add_argument('--reps', type=int, default=10, help='timed train() calls per trainer and setting')
    return ap.parse_args()


def make_trainer(args, captured):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl as cp, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    n, h = args.num_envs, args.horizon
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200.options(exact_infos=False))
    torch.manual_seed(1)
    policy = cleanrl.Policy(models.Default(vec.driver_env, hidden_size=128), fused_sample=True, seed=1).cuda()
    cfg = ppo_config(n, h, 'cuda', seed=1, cuda_graph=True)
    cfg.target_kl = 1e9
    cfg.manual_update = captured
    cfg.cuda_graph_train = captured
    cfg.cuda_graph_rollout = True
    data = cp.create(cfg, vec, policy)
    for _ in range(3):                      # eager call, then capture + first replay
        cp.evaluate(data)
        cp.train(data)
    cp.evaluate(data)                       # the rollout every timed call trains on
    return data


def adam_tensors(opt):
    return [opt.state[p][k] for p in opt.param_groups[0]['params'] for k in ('exp_avg', 'exp_avg_sq', 'step')]


class Snapshot:
    def __init__(self, data):
        from pufferlib_b200 import clean_pufferl as cp
        self.cp, self.data = cp, data
        self.params = [p.detach().clone() for p in data.policy.parameters()]
        self.adam = [t.clone() for t in adam_tensors(data.optimizer)]

    def restore(self):
        with torch.no_grad():
            for p, s in zip(self.data.policy.parameters(), self.params):
                p.copy_(s)
            for t, s in zip(adam_tensors(self.data.optimizer), self.adam):
                t.copy_(s)
        self.cp._invalidate_policy_cache(self.data)


def epoch_kls(data, snap):
    """The approx_kl each stop decision of one eager train() reads (epochs 0 .. E-2), from the snapshot."""
    from pufferlib_b200 import clean_pufferl as cp
    seen, orig = [], cp._KLStop.decide

    def spy(self, epoch, approx_kl=None, stats=None, row=0, rows=0):
        seen.append(float(approx_kl.detach()) if approx_kl is not None else float((stats[row, 4] / rows).float()))
        return orig(self, epoch, approx_kl=approx_kl, stats=stats, row=row, rows=rows)
    graph = data.config.cuda_graph_train
    cp._KLStop.decide, data.config.cuda_graph_train, data.config.target_kl = spy, False, 1e9
    try:
        snap.restore()
        cp.train(data)
    finally:
        cp._KLStop.decide, data.config.cuda_graph_train = orig, graph
    return seen


def main():
    args = parse_args()
    from pufferlib_b200 import clean_pufferl as cp
    torch.cuda.set_device(0)
    runs = {'autograd_eager': make_trainer(args, False), 'captured': make_trainer(args, True)}
    snaps = {k: Snapshot(d) for k, d in runs.items()}
    kls = {k: epoch_kls(d, snaps[k]) for k, d in runs.items()}
    out = dict(gpu=gpu_info(0), num_envs=args.num_envs, horizon=args.horizon, minibatches=4, epochs=4, reps=args.reps,
               statistic='median', epoch_kls=kls, method='CUDA events around train(), trainers alternated, parameters '
               'and Adam state restored before every call (outside the timed window)')
    for setting in ('never', 'after_epoch_1'):
        for k, d in runs.items():
            d.config.target_kl = 1e9 if setting == 'never' else 0.5 * (kls[k][0] + kls[k][1])
            snaps[k].restore()
            cp.train(d)                      # warm: the eager path's first call at this setting
        times, epochs = {k: [] for k in runs}, {k: set() for k in runs}
        for _ in range(args.reps):
            for k, d in runs.items():
                snaps[k].restore()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                cp.train(d)
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1))
                epochs[k].add(d.train_epochs_run)
        res = {}
        for k, d in runs.items():
            plan = cp.update_plan(d)
            res[k] = dict(train_ms=float(np.median(times[k])), train_ms_min_max=[min(times[k]), max(times[k])],
                          epochs_run=sorted(epochs[k]), target_kl=d.config.target_kl, engine=plan.engine,
                          capture=plan.capture, train_graph_state=d.train_graph_state)
        res['speedup'] = res['autograd_eager']['train_ms'] / res['captured']['train_ms']
        out[setting] = res
    for d in runs.values():
        cp.close(d)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
