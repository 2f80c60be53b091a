"""The multiagent ocean env on the device (PB_ENV_MULTIAGENT, two agent rows per env) + vectoriser vs the reference's own
trajectories (tests/golden/multiagent_*.npz) and vs the oracle at scale: bitwise obs, reward bits, terminals,
truncations, masks; exact per-agent infos; the per-agent statistics; and PPO on it (create / evaluate / train)."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
from multiagent_oracle import MultiagentSerial, info_rows
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.exceptions import APIUsageError
from pufferlib_b200.frameworks import cleanrl
from test_multiagent_cpu import MP_CASES, SERIAL_CASES

pytestmark = pytest.mark.gpu


def to_np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def make_vec(g, backend, **kw):
    n, w = int(g['num_envs']), int(g['num_workers'])
    if w:
        kw.update(num_workers=w, batch_size=n)
    return pvec.make(ocean.env_creator('multiagent'), num_envs=n, backend=backend, **kw)


def check_infos(infos):
    """The reference's info dicts: {1: {'score': int}, 2: {'score': int}}, python ints."""
    for i in infos:
        assert list(i) == [1, 2] and all(type(k) is int for k in i), i
        for a in (1, 2):
            assert list(i[a]) == ['score'] and type(i[a]['score']) is int, i


def run_case(g, backend, actions_on_device, bound=False):
    n, seed, h = int(g['num_envs']), int(g['seed']), int(g['horizon'])
    rows = 2 * n
    vec = make_vec(g, backend)
    assert vec.num_agents == vec.agents_per_batch == vec.num_envs == rows and vec.driver_env.num_agents == 2
    if bound:
        exp = clean_pufferl.Experience(rows * 8, 4, rows * 8, (1,), np.float32, ())
        vec.bind_rollout(exp)
    vec.async_reset(seed)
    got = []
    for t in range(h + 1):
        o, r, term, trunc, infos, ids, mask = vec.recv()
        assert np.array_equal(to_np(o).view(np.uint32), g['obs'][t].view(np.uint32)), f'obs step {t}'
        assert np.array_equal(to_np(r).view(np.uint32), g['rewards'][t].view(np.uint32)), f'reward bits step {t}'
        assert np.array_equal(to_np(term), g['terminals'][t]), f'terminals step {t}'
        assert np.array_equal(to_np(trunc), g['truncations'][t])
        assert np.array_equal(to_np(mask), g['masks'][t])
        assert np.array_equal(ids, np.arange(rows))
        check_infos(infos)
        got += info_rows(t, infos)
        if t < h:
            a = g['actions'][t]
            if bound:
                ad = torch.as_tensor(a, device='cuda')
                z = torch.zeros(rows, device='cuda')
                exp.store(o, z, ad, z, r, term, ids, mask)
                if exp.full:
                    exp.sort_training_data()
            vec.send(torch.as_tensor(a, device='cuda') if actions_on_device else a)
    assert np.array_equal(np.asarray(got, dtype=np.int64).reshape(-1, 4), g['infos'])
    vec.close()


@pytest.mark.parametrize('case', SERIAL_CASES + MP_CASES)
def test_multiagent_device_tensors(golden, case):
    run_case(golden(case), pvec.B200.options(exact_infos=True), actions_on_device=True)


@pytest.mark.parametrize('case', SERIAL_CASES + MP_CASES)
def test_multiagent_host_buffers(golden, case):
    """host_buffers=True: numpy in / numpy out like vector.Serial, infos equal to the reference's."""
    run_case(golden(case), pvec.B200.options(host_buffers=True), actions_on_device=False)


@pytest.mark.parametrize('case', SERIAL_CASES + MP_CASES)
def test_multiagent_bound_rollout(golden, case):
    """send() writing obs / reward / done rows straight into a bound Experience (row t*2N + 2e + a)."""
    run_case(golden(case), pvec.B200.options(exact_infos=True), actions_on_device=True, bound=True)


def test_multiagent_bound_rollout_rows(golden):
    """The bound rollout's rows are the golden's rows in arrival order, and a batch that is not a multiple of the agent
    rows is refused."""
    g = golden('multiagent_n5')
    n, rows = 5, 10
    vec = make_vec(g, pvec.B200)
    with pytest.raises(APIUsageError):
        vec.bind_rollout(clean_pufferl.Experience(36, 4, 36, (1,), np.float32, ()))     # 36 % 10 != 0
    h = 8
    exp = clean_pufferl.Experience(rows * h, 4, rows * h, (1,), np.float32, ())
    vec.bind_rollout(exp)
    vec.async_reset(int(g['seed']))
    for t in range(h):
        o, r, term, trunc, infos, ids, mask = vec.recv()
        z = torch.zeros(rows, device='cuda')
        exp.store(o, z, torch.as_tensor(g['actions'][t], device='cuda'), z, r, term, ids, mask)
        vec.send(torch.as_tensor(g['actions'][t], device='cuda'))
    assert np.array_equal(to_np(exp.obs).reshape(h, rows, 1), g['obs'][:h])
    assert np.array_equal(to_np(exp.rewards).reshape(h, rows), g['rewards'][:h])
    assert np.array_equal(to_np(exp.dones).reshape(h, rows), g['terminals'][:h].astype(np.float32))
    vec.close()


@pytest.mark.parametrize('case', SERIAL_CASES + MP_CASES)
def test_multiagent_episode_stats(golden, case):
    """episode_stats(): per-agent score means over the step-sends, the '1/score' / '2/score' keys of the reference's
    evaluate; one 32-byte read that clears."""
    g = golden(case)
    h = int(g['horizon'])
    vec = make_vec(g, pvec.B200)
    vec.async_reset(int(g['seed']))
    for t in range(h):
        vec.recv()
        vec.send(torch.as_tensor(g['actions'][t], device='cuda'))
    vec.recv()
    means, count = vec.episode_stats()
    ref = g['infos']
    assert count == len(ref) // 2
    assert set(means) == {'1/score', '2/score'}
    for a in (1, 2):
        assert means[f'{a}/score'] == ref[ref[:, 2] == a, 3].mean(), a
    assert vec.episode_stats() == ({}, 0)            # cleared
    vec.close()


def test_multiagent_pool_mode():
    """Pool mode (batch_size < num_envs counts envs): groups of batch_size envs, each returning 2 * batch_size agent rows
    round-robin, every env following the Serial oracle."""
    n, b, steps = 12, 4, 9
    vec = pvec.make(ocean.env_creator('multiagent'), num_envs=n, num_workers=3, batch_size=b,
                    backend=pvec.B200.options(exact_infos=True))
    assert isinstance(vec, pvec.B200Pool) and len(vec.groups) == 3
    assert vec.num_agents == 2 * n and vec.agents_per_batch == vec.num_envs == 2 * b
    oracles = [MultiagentSerial(b) for _ in range(3)]
    rng = np.random.default_rng(4)
    vec.async_reset(1)
    for o_ in oracles:
        o_.async_reset(1)
    for t in range(steps + 1):
        for k in range(3):
            o, r, d, tr, infos, ids, m = vec.recv()
            oo, orr, od, otr, oinf, _, om = oracles[k].recv()
            assert np.array_equal(ids, np.arange(2 * b * k, 2 * b * (k + 1)))
            assert np.array_equal(to_np(o), oo) and np.array_equal(to_np(r), orr) and np.array_equal(to_np(d), od)
            assert np.array_equal(to_np(m), om) and np.array_equal(to_np(tr), otr)
            assert infos == oinf, (t, k)
            a = rng.integers(0, 2, size=2 * b)
            vec.send(torch.as_tensor(a, device='cuda'))
            oracles[k].send(a)
    means, cnt = vec.episode_stats()
    assert cnt == 3 * b * ((steps + 1) // 2)
    vec.close()


def test_multiagent_matches_oracle_at_scale():
    """N = 16 384 envs (32 768 agent rows) against the oracle over 64 sends with a random action tape: rows bitwise,
    infos equal, the per-agent statistics equal to the infos' means."""
    n, steps = 16384, 64
    rng = np.random.default_rng(5)
    vec = pvec.make(ocean.env_creator('multiagent'), num_envs=n, backend=pvec.B200.options(exact_infos=True))
    ora = MultiagentSerial(n)
    vec.async_reset(1000)
    ora.async_reset(1000)
    sums, cnt = np.zeros(2), 0
    for t in range(steps + 1):
        o, r, term, trunc, infos, ids, mask = vec.recv()
        oo, orr, ot, otr, oinf, _, om = ora.recv()
        assert np.array_equal(to_np(o), oo), t
        assert np.array_equal(to_np(r).view(np.uint32), orr.view(np.uint32)), t
        assert np.array_equal(to_np(term), ot) and np.array_equal(to_np(trunc), otr) and np.array_equal(to_np(mask), om)
        assert infos == oinf, t
        for i in oinf:
            sums += (i[1]['score'], i[2]['score'])
        cnt += len(oinf)
        if t < steps:
            a = rng.integers(0, 2, size=2 * n)
            vec.send(torch.as_tensor(a, device='cuda') if t % 2 else a)
            ora.send(a)
    means, c = vec.episode_stats()
    assert c == cnt == n * (steps // 2)
    assert means == {'1/score': sums[0] / cnt, '2/score': sums[1] / cnt}
    vec.close()


def test_library_info_agents_and_refusals():
    """pb_env_get_info / pb_env_agents_per_env / the spaces come from the library; multiagent takes no parameters;
    the agent statistics read refuses single-agent kinds."""
    lib = _native.lib()
    cfg = _native.EnvConfig(kind=_native.ENV_KINDS['multiagent'], num_envs=6, device=0)
    h = C.c_void_p()
    _native.check(lib.pb_env_create(C.byref(cfg), C.byref(h)))
    info, agents = _native.EnvInfo(), C.c_int32()
    _native.check(lib.pb_env_get_info(h, C.byref(info)))
    _native.check(lib.pb_env_agents_per_env(h, C.byref(agents)))
    assert agents.value == 2 and info.num_envs == 6 and info.num_actions == 2 and info.obs_bytes == 4
    assert info.obs_ndim == 1 and info.obs_shape[0] == 1 and info.obs_low == 0 and info.obs_high == 1
    out = (C.c_double * 4)()
    _native.check(lib.pb_env_agent_stats_read(h, out, 1, None))
    assert list(out) == [0.0] * 4
    lib.pb_env_destroy(h)
    for ip, dp in (([1], []), ([0, 0, 0, 0, 0, 0, 0, 2], []), ([], [0.5]), ([], [0.0])):
        cfg = _native.EnvConfig(kind=_native.ENV_KINDS['multiagent'], num_envs=4, device=0,
                                iparam=(C.c_int32 * 8)(*(ip + [0] * (8 - len(ip)))))
        h = C.c_void_p()
        arr = (C.c_double * max(len(dp), 1))(*dp)
        assert lib.pb_env_create_ex(C.byref(cfg), arr, len(dp), C.byref(h)) == _native.PB_ERR_INVALID, (ip, dp)
        assert not h.value
    cfg = _native.EnvConfig(kind=_native.ENV_KINDS['bandit'], num_envs=4, device=0)
    h = C.c_void_p()
    _native.check(lib.pb_env_create(C.byref(cfg), C.byref(h)))
    _native.check(lib.pb_env_agents_per_env(h, C.byref(agents)))
    assert agents.value == 1
    assert lib.pb_env_agent_stats_read(h, out, 1, None) == _native.PB_ERR_INVALID
    lib.pb_env_destroy(h)

    vec = pvec.make(ocean.env_creator('multiagent'), num_envs=3, backend=pvec.B200)
    sp = vec.single_observation_space
    assert sp.shape == (1,) and sp.dtype == np.float32 and float(sp.low.min()) == 0 and float(sp.high.max()) == 1
    assert vec.single_action_space.n == 2 and vec.action_space.shape == (6,) and vec.observation_space.shape == (6, 1)
    with pytest.raises(APIUsageError):       # the first send checks all 2N actions
        vec.async_reset(0)
        vec.recv()
        vec.send(torch.zeros(3, dtype=torch.int64, device='cuda'))
    vec.close()
    with pytest.raises(APIUsageError):
        pvec.make(ocean.env_creator('multiagent'), env_args=[2], num_envs=2, backend=pvec.B200)


# -- PPO on multiagent -------------------------------------------------------------------------------------------------

N, H = 1024, 32


def make_config(**kw):
    cfg = dict(seed=1, torch_deterministic=True, env='ocean', batch_size=2 * N * H, bptt_horizon=8,
               minibatch_size=2 * N * H // 4, cpu_offload=False, device='cuda', compile=False, learning_rate=3e-3,
               gamma=0.95, gae_lambda=0.9, update_epochs=2, norm_adv=True, clip_coef=0.2, clip_vloss=True,
               vf_clip_coef=0.2, vf_coef=0.5, ent_coef=0.01, max_grad_norm=0.5, target_kl=None, anneal_lr=False,
               total_timesteps=10 ** 9, cuda_graph=True)
    cfg.update(kw)
    return pufferlib_b200.namespace(**cfg)


def run_learning(seed, iters):
    """models.Default through create / evaluate / train with cuda_graph=True -> (first iteration whose rollout had both
    agents' score >= 0.9, or None; [(1/score, 2/score)] per iteration)."""
    torch.manual_seed(seed)
    vec = pvec.make(ocean.env_creator('multiagent'), num_envs=N, backend=pvec.B200)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=seed).cuda()
    data = clean_pufferl.create(make_config(seed=seed), vec, pol)
    history, first = [], None
    for it in range(iters):
        clean_pufferl.evaluate(data)
        s = (data.stats.get('1/score'), data.stats.get('2/score'))
        history.append(s)
        if None not in s and min(s) >= 0.9:
            first = it
            break
        clean_pufferl.train(data)
    assert data.graph_state == 2 or (first is not None and first < 2)      # the captured rollout ran
    clean_pufferl.close(data)
    return first, history


# iterations (evaluate + train) allowed: >= 2x the worst of seeds 1, 2, 3 on an H100 (DESIGN.md §4)
BUDGET = 10


def test_multiagent_learns():
    first, history = run_learning(seed=1, iters=BUDGET)
    print(f'[multiagent learning] passed at iteration {first}; last scores {history[-3:]}', flush=True)
    assert first is not None, history


def test_lstm_rollout_per_agent_state_matches_cudnn():
    """RecurrentPolicy(LSTMWrapper(Default), fused_sample=True, fused_update=True) through one evaluate + train on
    multiagent: the LSTM state is indexed per agent row (agents 1 and 2 of an env see different observations, so their
    states differ).  Replaying the fused rollout's actions through the cuDNN RecurrentPolicy with the same weights gives its
    logprobs within 1e-5 and its final state within TOL_STATE."""
    n, h = 256, 16
    rows = 2 * n
    torch.manual_seed(3)
    vec = pvec.make(ocean.env_creator('multiagent'), num_envs=n, backend=pvec.B200)
    env = vec.driver_env
    net = models.LSTMWrapper(env, models.Default(env), input_size=128, hidden_size=128)
    init = {k: v.clone() for k, v in net.state_dict().items()}
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=7, fused_update=True).cuda()
    cfg = make_config(batch_size=rows * h, minibatch_size=rows * h // 2, bptt_horizon=8, cuda_graph=False)
    data = clean_pufferl.create(cfg, vec, pol)
    clean_pufferl.evaluate(data)
    x = data.experience
    assert tuple(x.lstm_h.shape) == (1, rows, 128)
    actions, logprobs = x.actions.clone().view(h, rows), x.logprobs.clone().view(h, rows)
    state_h, state_c = x.lstm_h.clone(), x.lstm_c.clone()
    obs = x.obs.clone().view(h, rows, 1)
    assert not torch.equal(state_h[:, 0::2], state_h[:, 1::2])
    clean_pufferl.train(data)
    assert data.train_recurrent_path == 'fused'
    clean_pufferl.close(data)

    ref = models.LSTMWrapper(env, models.Default(env), input_size=128, hidden_size=128)
    ref.load_state_dict(init)
    ref = cleanrl.RecurrentPolicy(ref).cuda()
    hs = torch.zeros(1, rows, 128, device='cuda')
    cs = torch.zeros(1, rows, 128, device='cuda')
    errs = {'logprob': 0.0}
    with torch.no_grad():
        for t in range(h):
            _, lp, _, _, (hs, cs) = ref(obs[t], (hs, cs), actions[t])
            errs['logprob'] = max(errs['logprob'], float((lp - logprobs[t]).abs().max()))
    errs['h'] = float((hs - state_h).abs().max())
    errs['c'] = float((cs - state_c).abs().max())
    print('[multiagent lstm] fused rollout vs cuDNN, max abs err', {k: f'{e:.2e}' for k, e in errs.items()}, flush=True)
    assert errs['logprob'] <= 1e-5, errs
    assert errs['h'] <= TOL_STATE and errs['c'] <= TOL_STATE, errs


# the fused step runs its products on TF32 tensor cores (operands rounded to nearest TF32), cuDNN on its own TF32 path, and
# the state carries the difference through the 16 steps: the rollout bound of tests/test_gpu_policy_lstm.py.  Observed on
# an H100 (80GB HBM3, 400 W power limit): logprob 6.0e-7, h 1.3e-4, c 2.5e-4
TOL_STATE = 5e-4
