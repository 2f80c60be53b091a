"""The fused recurrent rollout step (pb_policy_lstm_sample, csrc/policy_lstm.cu) behind
cleanrl.RecurrentPolicy(models.LSTMWrapper(models.Default), fused_sample=True).

Kernel outputs are checked against an fp64 restatement that models the kernel's operand rounding (every tensor-core operand
rounded to nearest TF32, cvt.rna); sampled actions against the inverse CDF of the counter-based uniform; rollouts replay
bit-exactly through the oracles.  Reference loop: reference clean_pufferl.py:84-124 (state carry :100-105)."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models, spaces
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from util_gpu import off_boundary_mismatches, rna

gpu = pytest.mark.gpu
TOL = 2e-4              # per-step kernel outputs vs the fp64 restatement
TOL_ROLLOUT = 5e-4      # the same after up to 128 recurrent steps (the fp64 state is carried, not the kernel's)


def cpu(x):
    return x.detach().cpu().numpy()


def reference_step(net, x, h, c):
    """fp64 restatement of one pb_policy_lstm_sample step -> (h', c', out [m, 8 or 16])."""
    inner, rnn = net.policy, net.recurrent
    x = x.reshape(x.shape[0], -1)
    e = torch.relu(rna(x) @ rna(inner.encoder.weight).t() + inner.encoder.bias.double())
    z = (rna(e) @ rna(rnn.weight_ih_l0).t() + rna(h) @ rna(rnn.weight_hh_l0).t()
         + (rnn.bias_ih_l0 + rnn.bias_hh_l0).double())
    i, f, g, o = z.chunk(4, 1)
    c2 = torch.sigmoid(f) * c.double() + torch.sigmoid(i) * torch.tanh(g)
    h2 = torch.sigmoid(o) * torch.tanh(c2)
    w_cat, b_cat = inner.head_matrix()
    return h2, c2, rna(h2) @ rna(w_cat).t() + b_cat.double()


def fake_env(obs_shape, n_act, dtype=np.float32):
    return types.SimpleNamespace(single_observation_space=spaces.Box(0, 1, obs_shape, dtype),
                                 single_action_space=spaces.Discrete(n_act))


def sharpen(net):
    """Non-trivial heads and biases: the default init gives almost uniform policies and zero LSTM biases."""
    with torch.no_grad():
        net.policy.decoder.weight.mul_(20.0)
        net.policy.value_head.weight.mul_(3.0)
        for name, p in net.recurrent.named_parameters():
            if 'bias' in name:
                p.uniform_(-0.5, 0.5)


def make_policy(obs_shape, n_act, hidden=128, layers=1, dtype=np.float32, seed=11):
    torch.manual_seed(0)
    env = fake_env(obs_shape, n_act, dtype)
    net = models.LSTMWrapper(env, models.Default(env, hidden_size=hidden), input_size=hidden, hidden_size=hidden,
                             num_layers=layers)
    sharpen(net)
    return cleanrl.RecurrentPolicy(net, fused_sample=True, seed=seed).cuda()


def make_config(n, h, **kw):
    cfg = dict(seed=1, torch_deterministic=True, env='squared', batch_size=n * h, bptt_horizon=8, minibatch_size=n * h // 2,
               cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
               update_epochs=2, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5,
               ent_coef=0.01, max_grad_norm=0.5, target_kl=None, anneal_lr=False, total_timesteps=10 ** 9)
    cfg.update(kw)
    return pufferlib_b200.namespace(**cfg)


def test_unsupported_shapes_are_refused_before_any_launch():
    """PB_ERR_UNSUPPORTED for > 128 features, LSTM sizes other than 128 and more than 15 actions (no device needed: the
    checks come before any CUDA call)."""
    lib = _native.lib()
    p = C.c_void_p(256)

    def call(feats=49, size=128, hidden=128, n_act=8):
        return lib.pb_policy_lstm_sample(p, feats, feats, p, p, p, p, p, p, p, 128, p, 128, 4, size, hidden, n_act,
                                         C.c_uint64(0), None, None, p, p, p, None, None)
    assert call(feats=129) == _native.PB_ERR_UNSUPPORTED
    assert call(size=64) == _native.PB_ERR_UNSUPPORTED
    assert call(hidden=256) == _native.PB_ERR_UNSUPPORTED
    assert call(n_act=16) == _native.PB_ERR_UNSUPPORTED
    assert lib.pb_policy_lstm_sample(p, 49, 49, p, p, p, p, p, p, p, 128, p, 128, 0, 128, 128, 8, C.c_uint64(0), None,
                                     None, p, p, p, None, None) == _native.PB_OK      # m = 0: nothing to do


@gpu
@pytest.mark.parametrize('n_act', [4, 8, 15])
@pytest.mark.parametrize('m', [1, 64, 1000, 16384])
@pytest.mark.parametrize('feats', [49, 128])
def test_kernel_matches_fp64(feats, m, n_act):
    """h', c', value, logprob and entropy vs the fp64 restatement; actions vs the inverse CDF off CDF boundaries; the counter
    advances by one; guard rows around h / c / the output rows stay untouched.  Largest errors observed over all 24 cases
    (H100 80GB HBM3, 400 W power limit; the kernel is deterministic): value 1.44e-4 (the value head is scaled by 3),
    c 9.3e-5, h 5.1e-5, logprob 1.9e-5, entropy 9.2e-7; bound TOL = 2e-4."""
    pol = make_policy((feats,), n_act)
    gen = torch.Generator(device='cuda').manual_seed(1000 * feats + m + n_act)
    x = torch.rand(m, feats, device='cuda', generator=gen) * 2 - 1
    h0 = torch.randn(m, 128, device='cuda', generator=gen) * 0.5
    c0 = torch.randn(m, 128, device='cuda', generator=gen)
    G = 32
    hbuf = torch.full((m + 2 * G, 128), 7.0, device='cuda')
    cbuf = torch.full((m + 2 * G, 128), 7.0, device='cuda')
    hbuf[G:G + m], cbuf[G:G + m] = h0, c0
    vbuf = torch.full((m + 2 * G,), 7.0, device='cuda')
    lbuf = torch.full((m + 2 * G,), 7.0, device='cuda')
    abuf = torch.full((m + 2 * G,), -7, dtype=torch.int64, device='cuda')
    h, c = hbuf[G:G + m].unsqueeze(0), cbuf[G:G + m].unsqueeze(0)
    with torch.no_grad():
        a, lp, ent, v, (h1, c1) = pol(x, (h, c), out=(vbuf[G:G + m], lbuf[G:G + m], abuf[G:G + m]))
    torch.cuda.synchronize()
    assert h1.data_ptr() == h.data_ptr() and c1.data_ptr() == c.data_ptr()          # updated in place
    assert int(pol._counter[0]) == 1
    with torch.no_grad():
        h2, c2, out = reference_step(pol.policy, x, h0, c0)
    logits, value = out[:, :n_act], out[:, n_act]
    norm = logits - logits.logsumexp(-1, keepdim=True)
    errs = {'h': float((hbuf[G:G + m].double() - h2).abs().max()), 'c': float((cbuf[G:G + m].double() - c2).abs().max()),
            'value': float((vbuf[G:G + m].double() - value).abs().max()),
            'logprob': float((lbuf[G:G + m].double() - norm.gather(-1, abuf[G:G + m].view(-1, 1)).squeeze(-1)).abs().max()),
            'entropy': float((ent.double() + (norm.exp() * norm).sum(-1)).abs().max())}
    print(f'[lstm-kernel] F={feats} m={m} n_act={n_act} max err', {k: f'{e:.2e}' for k, e in errs.items()}, flush=True)
    assert all(e < TOL for e in errs.values()), errs
    assert off_boundary_mismatches(cpu(abuf[G:G + m]), logits, pol._seed, 0) == 0
    for buf, fill in ((hbuf, 7.0), (cbuf, 7.0), (vbuf, 7.0), (lbuf, 7.0), (abuf, -7)):
        assert bool((buf[:G] == fill).all()) and bool((buf[G + m:] == fill).all())
    assert a.data_ptr() == abuf[G:].data_ptr() and v.data_ptr() == vbuf[G:].data_ptr()


@gpu
def test_pool_slice_is_updated_in_place():
    """A slice lstm_h[:, lo:hi] (one pool group) is updated in place; every other row is bit-unchanged."""
    pol = make_policy((128,), 4)
    n, lo, hi = 256, 64, 192
    gen = torch.Generator(device='cuda').manual_seed(5)
    lstm_h = torch.randn(1, n, 128, device='cuda', generator=gen) * 0.5
    lstm_c = torch.randn(1, n, 128, device='cuda', generator=gen)
    h_before, c_before = lstm_h.clone(), lstm_c.clone()
    x = torch.rand(hi - lo, 128, device='cuda', generator=gen)
    with torch.no_grad():
        _, _, _, v, (h1, c1) = pol(x, (lstm_h[:, lo:hi], lstm_c[:, lo:hi]))
        h2, c2, out = reference_step(pol.policy, x, h_before[0, lo:hi], c_before[0, lo:hi])
    torch.cuda.synchronize()
    assert h1.data_ptr() == lstm_h[:, lo:hi].data_ptr()
    for now, before in ((lstm_h, h_before), (lstm_c, c_before)):
        assert torch.equal(now[:, :lo], before[:, :lo]) and torch.equal(now[:, hi:], before[:, hi:])
    assert float((lstm_h[0, lo:hi].double() - h2).abs().max()) < TOL
    assert float((lstm_c[0, lo:hi].double() - c2).abs().max()) < TOL
    assert float((v.double() - out[:, 4]).abs().max()) < TOL


@gpu
@pytest.mark.parametrize('env,n,h', [('squared', 64, 128), ('breakout', 256, 64)])
def test_fused_recurrent_rollout_replays(env, n, h):
    """evaluate() with the fused recurrent step: the env rows replay bit-exactly through the oracle with the stored actions,
    the fp64 recurrence on the stored observations gives the stored values / logprobs and the final lstm_h / lstm_c, the
    actions are the inverse CDF of each step's uniforms, and train() afterwards gives finite losses.  Largest errors
    observed (H100 80GB HBM3): value 9.9e-5, logprob 1.5e-5, lstm_h 1.5e-5, lstm_c 2.4e-5; bound TOL_ROLLOUT = 5e-4."""
    check_recurrent_rollout_replays(env, n, h)


def rollout_oracle(env, n):
    """The oracle vectoriser of env kind `env` over n envs."""
    from oracle.envs import OracleVec
    from oracle.ocean import OceanSerial
    from oracle.squared import SquaredSerial
    if env == 'squared':
        return SquaredSerial(n)
    if env == 'breakout':
        return OracleVec('breakout', n)
    return OceanSerial(env, n)


def check_recurrent_rollout_replays(env, n, h):
    """The body of test_fused_recurrent_rollout_replays for env kind `env`, n envs, h steps."""
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
    sharpen(net)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=3).cuda()
    data = clean_pufferl.create(make_config(n, h, env=env), vec, pol)
    assert data.fused_rows
    clean_pufferl.evaluate(data)
    exp = data.experience
    ora = rollout_oracle(env, n)
    ora.async_reset(1)
    obs_shape = tuple(vec.single_observation_space.shape)
    acts, obs = cpu(exp.actions).reshape(h, n), cpu(exp.obs).reshape(h, n, *obs_shape)
    rew, done = cpu(exp.rewards).reshape(h, n), cpu(exp.dones).reshape(h, n)
    for t in range(h):
        o, r, d, _, _, _, _ = ora.recv()
        assert np.array_equal(o, obs[t]), t
        assert np.array_equal(np.asarray(r, np.float32).view(np.uint32), rew[t].view(np.uint32)), t
        assert np.array_equal(np.asarray(d).astype(np.float32), done[t]), t
        ora.send(acts[t])
    n_act = vec.single_action_space.n
    hr = torch.zeros(n, 128, dtype=torch.float64, device='cuda')
    cr = torch.zeros_like(hr)
    dv = dl = 0.0
    bad = 0
    with torch.no_grad():
        for t in range(h):
            hr, cr, out = reference_step(net, exp.obs[t * n:(t + 1) * n], hr, cr)
            logits = out[:, :n_act]
            norm = logits - logits.logsumexp(-1, keepdim=True)
            dv = max(dv, float((exp.values[t * n:(t + 1) * n].double() - out[:, n_act]).abs().max()))
            lp = norm.gather(-1, exp.actions[t * n:(t + 1) * n].view(-1, 1)).squeeze(-1)
            dl = max(dl, float((exp.logprobs[t * n:(t + 1) * n].double() - lp).abs().max()))
            bad += off_boundary_mismatches(acts[t], logits, pol._seed, t)
    dh = float((exp.lstm_h[0].double() - hr).abs().max())
    dc = float((exp.lstm_c[0].double() - cr).abs().max())
    print(f'[lstm-rollout] {env} n={n} h={h}: max err value {dv:.2e} logprob {dl:.2e} lstm_h {dh:.2e} lstm_c {dc:.2e}',
          flush=True)
    assert max(dv, dl, dh, dc) < TOL_ROLLOUT, (dv, dl, dh, dc)
    assert bad == 0, bad
    assert int(pol._counter[0]) == h
    clean_pufferl.train(data)
    assert np.isfinite(data.losses.policy_loss) and np.isfinite(data.losses.value_loss)
    clean_pufferl.close(data)


@gpu
def test_graphed_recurrent_rollout_matches_eager():
    """A captured rollout with the fused recurrent step replays the computation of the eager loop: same seeds and config,
    rollout graph on vs off (the recurrent update is eager in both).  As in test_graphed_training_matches_eager_training,
    the comparison is made before sampling amplifies last-bit parameter differences of the updates: the first rollout is
    identical, the captured one (iteration 1) and the first replay (iteration 2) agree on nearly every action."""
    n, h = 64, 32
    acts, states = {}, {}
    for mode in ('eager', 'graph'):
        vec = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200)
        torch.manual_seed(0)
        net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
        sharpen(net)
        pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=7).cuda()
        g = mode == 'graph'
        data = clean_pufferl.create(make_config(n, h, env='breakout', cuda_graph=True, cuda_graph_rollout=g), vec, pol)
        acts[mode], states[mode] = [], []
        for it in range(3):
            clean_pufferl.evaluate(data)
            acts[mode].append(cpu(data.experience.actions).copy())
            states[mode].append(data.experience.lstm_h.detach().clone())
            clean_pufferl.train(data)
            assert np.isfinite(data.losses.policy_loss)
        assert data.graph_replays == (2 if g else 0)
        assert int(pol._counter[0]) == 3 * h
        clean_pufferl.close(data)
    agree = [float((a == b).mean()) for a, b in zip(acts['eager'], acts['graph'])]
    dh = [float((a - b).abs().max()) for a, b in zip(states['eager'], states['graph'])]
    print('[lstm-graph] action agreement', agree, 'max |lstm_h diff|', dh, flush=True)
    assert agree[0] == 1.0 and dh[0] == 0.0, (agree, dh)
    assert agree[1] > 0.9995 and agree[2] > 0.98, (agree, dh)


@gpu
@pytest.mark.parametrize('kind', ['hidden64', 'two_layers', 'uint8_obs'])
def test_unsupported_models_take_the_unfused_path(kind):
    """fused_sample=True with a model the kernel does not cover computes exactly what fused_sample=False computes."""
    n = 96
    if kind == 'uint8_obs':             # snake's observations: 16 x 16 uint8
        pol = make_policy((16, 16), 4, dtype=np.uint8)
        x = torch.randint(0, 4, (n, 16, 16), dtype=torch.uint8, device='cuda')
    else:
        pol = make_policy((49,), 8, hidden=64 if kind == 'hidden64' else 128, layers=2 if kind == 'two_layers' else 1)
        x = torch.rand(n, 49, device='cuda')
    rnn = pol.policy.recurrent
    gen = torch.Generator(device='cuda').manual_seed(9)
    state = (torch.randn(rnn.num_layers, n, rnn.hidden_size, device='cuda', generator=gen),
             torch.randn(rnn.num_layers, n, rnn.hidden_size, device='cuda', generator=gen))
    res = {}
    for fused in (False, True):
        pol.fused_sample = fused
        torch.manual_seed(123)
        with torch.no_grad():
            a, lp, ent, v, (h1, c1) = pol(x, (state[0].clone(), state[1].clone()))
        res[fused] = [t.detach().clone() for t in (a, lp, ent, v, h1, c1)]
    assert pol._counter is None                       # the kernel never ran
    for u, w in zip(res[False], res[True]):
        assert torch.equal(u, w)
