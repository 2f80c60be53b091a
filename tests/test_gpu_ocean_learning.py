"""The ocean test envs doing what they are for: end-to-end PPO runs (clean_pufferl create / evaluate / train with
cuda_graph=True) that show what each policy can learn.

  memory      RecurrentPolicy(LSTMWrapper(Default), fused_sample, fused_update) recalls the digits (score >= 0.9) on
              the fused BPTT update; Default alone stays at chance (0.25 at L = 2: its obs on the answer ticks is 0).
  password    Default finds the constant password (score >= 0.9).
  stochastic  Default plays action 0 with probability within 0.05 of p, averaged over the last 20 rollouts of a fixed
              run: a single rollout's share swings by about +-0.15 from one iteration to the next (the reward depends on
              the share so far, so each update overshoots), at any learning rate tried.
  bandit      Default pulls the winning arm (6 of 10) at least 90% of the time.

Each case runs on one seed with an iteration budget of at least twice the worst of three seeds measured on an H100
(DESIGN.md §4); `run_case` is also what tests/experimental/measure_ocean_learning.py calls."""
import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
from pufferlib_b200 import clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl

pytestmark = pytest.mark.gpu

N, H = 1024, 32


def make_config(**kw):
    cfg = dict(seed=1, torch_deterministic=True, env='ocean', batch_size=N * H, bptt_horizon=8,
               minibatch_size=N * H // 4, cpu_offload=False, device='cuda', compile=False, learning_rate=3e-3,
               gamma=0.95, gae_lambda=0.9, update_epochs=2, norm_adv=True, clip_coef=0.2, clip_vloss=True,
               vf_clip_coef=0.2, vf_coef=0.5, ent_coef=0.01, max_grad_norm=0.5, target_kl=None, anneal_lr=False,
               total_timesteps=10 ** 9, cuda_graph=True)
    cfg.update(kw)
    return pufferlib_b200.namespace(**cfg)


# per-case settings over make_config
OVERRIDES = {'stochastic': dict(learning_rate=1e-3)}
STOCHASTIC_WINDOW = 20


def metric(case, data):
    """The quantity each case is judged by, from the last rollout."""
    x = data.experience
    if case in ('memory_lstm', 'memory_mlp', 'password'):
        return data.stats.get('score')
    a = x.actions.float()
    if case == 'stochastic':
        return float((a == 0).float().mean())
    return float((a == 6).float().mean())


def passed(case, m, p=0.7):
    if m is None:
        return False
    if case == 'stochastic':
        return abs(m - p) <= 0.05
    return m >= 0.9


def first_pass(case, history):
    """First iteration whose rollout passed; for stochastic, the last iteration if the mean share of the last
    STOCHASTIC_WINDOW rollouts passed, else None."""
    if case == 'stochastic':
        tail = history[-STOCHASTIC_WINDOW:]
        return len(history) - 1 if len(tail) == STOCHASTIC_WINDOW and passed(case, float(np.mean(tail))) else None
    ok = [passed(case, m) for m in history]
    return ok.index(True) if True in ok else None


def run_case(case, seed, iters, stop_early=True):
    """-> (first iteration at which the metric passed, or None; the metric per iteration; paths record).  stop_early:
    stop at the first rollout that passed (not for stochastic, which runs all `iters`)."""
    stop_early = stop_early and case != 'stochastic'
    kind = case.split('_')[0]
    torch.manual_seed(seed)
    vec = pvec.make(ocean.env_creator(kind), num_envs=N, backend=pvec.B200)
    env = vec.driver_env
    if case == 'memory_lstm':
        net = models.LSTMWrapper(env, models.Default(env), input_size=128, hidden_size=128)
        pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=seed, fused_update=True).cuda()
    else:
        pol = cleanrl.Policy(models.Default(env), fused_sample=True, seed=seed).cuda()
    data = clean_pufferl.create(make_config(seed=seed, **OVERRIDES.get(case, {})), vec, pol)
    history, record = [], {}
    for it in range(iters):
        clean_pufferl.evaluate(data)
        m = metric(case, data)
        history.append(m)
        if stop_early and passed(case, m):
            break
        clean_pufferl.train(data)
        record = dict(minibatch_form=data.train_minibatch_path,
                      recurrent_path=getattr(data, 'train_recurrent_path', None),
                      update=('hand-written' if getattr(data, 'manual_update', None) is not None else 'autograd'),
                      graph_state=data.train_graph_state)
    clean_pufferl.close(data)
    return first_pass(case, history), history, record


# iterations (evaluate + train) allowed per case: >= 2x the worst of seeds 1, 2, 3 on an H100 (DESIGN.md §4); stochastic
# always runs its fixed 120
BUDGET = {'memory_lstm': 32, 'password': 20, 'stochastic': 120, 'bandit': 20}


@pytest.mark.parametrize('case', ['memory_lstm', 'password', 'stochastic', 'bandit'])
def test_ocean_learns(case):
    first, history, record = run_case(case, seed=1, iters=BUDGET[case])
    print(f'[ocean learning] {case}: passed at iteration {first}; {record}; last metrics {history[-3:]}', flush=True)
    assert first is not None, (case, history, record)
    if case == 'memory_lstm':
        assert record['recurrent_path'] == 'fused' and record['minibatch_form'] == 'segments', record
        assert record['graph_state'] == 2, record


def test_memory_mlp_stays_at_chance():
    """The MLP sees 0 on the answer ticks: it cannot beat chance (0.25 at L = 2) however long it trains."""
    _, history, record = run_case('memory_mlp', seed=1, iters=60, stop_early=False)
    tail = [m for m in history[-10:] if m is not None]
    print(f'[ocean learning] memory_mlp: {record}; last metrics {tail[-3:]}', flush=True)
    assert tail and max(tail) <= 0.35, tail
