"""breakout_pixels on the device against its oracle (oracle/breakout_pixels.py: the breakout oracle's game drawn by the
scalar C restatement of oracle/SPEC_BREAKOUT_PIXELS.md): bit-exact
(4, 84, 84) frame stacks, reward bits, terminals and EpisodeStats infos through every vectoriser mode, the same game as the
`breakout` kind, and models.Convolutional trained on it through create / evaluate / train with the rollout and the
update captured."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.exceptions import APIUsageError
from pufferlib_b200.frameworks import cleanrl
from oracle.breakout_pixels import BreakoutPixelsVec

pytestmark = pytest.mark.gpu

KIND = 'breakout_pixels'
SHAPE = (4, 84, 84)
ROW = 4 * 84 * 84


def cpu(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def tape(h, n, seed):
    # FIRE-heavy, so balls launch early, bricks fall and lives are lost within a few hundred steps
    return np.random.default_rng(seed).choice(4, size=(h, n), p=[0.2, 0.3, 0.25, 0.25]).astype(np.int64)


def oracle(n, max_ticks=None, offset=0):
    return BreakoutPixelsVec(n, env_index_offset=offset, iparam=[max_ticks] if max_ticks else [])


def kwargs_of(max_ticks):
    return {'max_ticks': max_ticks} if max_ticks else {}


def check_step(t, got, want, infos=True):
    o, r, term, trunc, inf, _, mask = got
    oo, orr, ot, _, oinf, _, _ = want
    o = cpu(o)
    if not np.array_equal(o, oo):
        bad = np.nonzero((o != oo).reshape(len(oo), -1).any(1))[0]
        raise AssertionError(f'step {t}: frames differ in envs {bad[:8]} ({len(bad)} envs)')
    assert np.array_equal(cpu(r).view(np.uint32), orr.view(np.uint32)), f'step {t}: reward bits differ'
    assert np.array_equal(cpu(term), ot), f'step {t}: terminals differ'
    assert not cpu(trunc).any() and cpu(mask).all()
    if infos:
        assert len(inf) == len(oinf), t
        for a, b in zip(inf, oinf):
            assert a['episode_length'] == b['episode_length'] and a['score'] == b['score'], t
            assert np.isclose(a['episode_return'], b['episode_return'], rtol=1e-12, atol=0), t


def compare_run(n, h, seed, max_ticks=None, offset=0, bound=False, host_buffers=False, infos=True, **make_kw):
    """Device vs oracle, every row of h steps (+ the reset row); -> (episodes ended, bricks hit)."""
    vec = pvec.make(ocean.env_creator(KIND), env_kwargs=kwargs_of(max_ticks), num_envs=n,
                    backend=pvec.B200.options(exact_infos=infos, env_index_offset=offset, host_buffers=host_buffers),
                    **make_kw)
    ora = oracle(n, max_ticks, offset)
    acts = tape(h, n, seed)
    vec.async_reset(seed)
    ora.async_reset(seed)
    exp = None
    if bound:
        rows = 8
        exp = clean_pufferl.Experience(n * rows, 4, n * rows, SHAPE, np.uint8, ())
        vec.bind_rollout(exp)
    eps = bricks = 0
    for t in range(h + 1):
        got = vec.recv()
        want = ora.recv()
        check_step(t, got, want, infos)
        eps += int(want[2].sum())
        bricks += int((want[1] > 0).sum())
        if t < h:
            a = torch.as_tensor(acts[t], device='cuda')
            if bound:
                z = torch.zeros(n, device='cuda')
                exp.store(got[0], z, a, z, got[1], got[2], got[5], got[6])
                if exp.full:
                    exp.sort_training_data()
            vec.send(a)
            ora.send(acts[t])
    vec.close()
    ora.close()
    return eps, bricks


# ---- 1. device vs oracle ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 5, 33, 263])
@pytest.mark.parametrize('seed', [3, 71])
def test_vs_oracle_short_episodes(n, seed):
    """60-tick episodes: many reset rows (all four slots the first frame) and infos."""
    eps, _ = compare_run(n, 200, seed + n, max_ticks=60)
    assert eps >= 3 * n


@pytest.mark.parametrize('n', [1, 5, 33])
def test_vs_oracle_default_params(n):
    """The default max_ticks over 600 steps: bricks fall, lives are lost, the ball crosses every brick row."""
    eps, bricks = compare_run(n, 600, 11 + n)
    assert bricks > 0


def test_vs_oracle_4096():
    eps, bricks = compare_run(4096, 40, 5, max_ticks=25, infos=False)
    assert eps > 0


def test_vs_oracle_env_index_offset():
    compare_run(16, 150, 9, max_ticks=50, offset=1000)
    compare_run(263, 60, 2, offset=12345)


@pytest.mark.parametrize('n', [5, 33])
def test_bound_rollout_rows(n):
    """Step outputs written straight into Experience rows, and the carry-over across rollout boundaries."""
    compare_run(n, 70, 5, max_ticks=30, bound=True)


def test_host_buffers():
    compare_run(33, 80, 6, max_ticks=30, host_buffers=True)


def test_num_workers():
    """num_workers: breakout_pixels keys its RNG by global env index, so the worker split cannot change any row."""
    compare_run(32, 80, 8, max_ticks=40, num_workers=2)


@pytest.mark.parametrize('groups', [2, 4])
def test_pool_mode(groups):
    """batch_size < num_envs: groups returned round-robin, every env's rows equal to the oracle's."""
    n, h = 64, 60
    b = n // groups
    vec = pvec.make(ocean.env_creator(KIND), env_kwargs={'max_ticks': 25}, num_envs=n, backend=pvec.B200, batch_size=b)
    assert isinstance(vec, pvec.B200Pool)
    ora = oracle(n, 25)
    acts = tape(h, n, 4)
    vec.async_reset(7)
    ora.async_reset(7)
    for t in range(h):
        oo, orr, ot, _, _, _, _ = ora.recv()
        for g in range(groups):
            o, r, term, _, _, ids, _ = vec.recv()
            lo, hi = g * b, (g + 1) * b
            assert np.array_equal(ids, np.arange(lo, hi))
            assert np.array_equal(cpu(o), oo[lo:hi]) and np.array_equal(cpu(r), orr[lo:hi]), (t, g)
            assert np.array_equal(cpu(term), ot[lo:hi]), (t, g)
            vec.send(torch.as_tensor(acts[t, lo:hi], device='cuda'))
        ora.send(acts[t])
    vec.close()


# ---- 2. the same game as `breakout` ----------------------------------------------------------------------------------
@pytest.mark.parametrize('max_ticks', [None, 45])
def test_same_game_as_breakout(max_ticks):
    """Same seed and tape: rewards, terminals and the infos (score = (120 - left) / 120) equal to breakout's bit for bit."""
    n, h = 64, 600
    vecs = [pvec.make(ocean.env_creator(k), env_kwargs=kwargs_of(max_ticks), num_envs=n,
                      backend=pvec.B200.options(exact_infos=True)) for k in ('breakout', KIND)]
    acts = tape(h, n, 13)
    for v in vecs:
        v.async_reset(13)
    eps = hits = 0
    for t in range(h + 1):
        (_, r0, t0, _, i0, _, _), (_, r1, t1, _, i1, _, _) = (v.recv() for v in vecs)
        assert np.array_equal(cpu(r0).view(np.uint32), cpu(r1).view(np.uint32)), t
        assert np.array_equal(cpu(t0), cpu(t1)) and i0 == i1, t
        eps += len(i0)
        hits += int((cpu(r0) > 0).sum())
        if t < h:
            for v in vecs:
                v.send(torch.as_tensor(acts[t], device='cuda'))
    assert (eps > 0) if max_ticks else (hits > 0), (hits, eps)      # short episodes end before a brick falls
    for v in vecs:
        v.close()


def test_spaces_and_info():
    vec = pvec.make(ocean.env_creator(KIND), num_envs=2, backend=pvec.B200)
    sp = vec.single_observation_space
    assert sp.shape == SHAPE and sp.dtype == np.uint8 and float(sp.low.min()) == 0 and float(sp.high.max()) == 255
    assert vec.single_action_space.n == 4 and vec.obs_bytes == ROW
    assert not vec.fused_rollout_ok(None, None)     # the persistent rollout kernel is breakout + models.Default only
    vec.close()
    with pytest.raises(APIUsageError):
        pvec.make(ocean.env_creator(KIND), env_kwargs={'max_ticks': 70000}, num_envs=2, backend=pvec.B200)


# ---- 3. invalid calls ------------------------------------------------------------------------------------------------
def test_misaligned_obs_refused_before_launch():
    """The bulk copies need 16-byte aligned rows: a misaligned obs pointer or stride is refused and nothing runs."""
    lib = _native.lib()
    n = 4
    cfg = _native.EnvConfig(kind=_native.ENV_KINDS[KIND], num_envs=n, device=0)
    h = C.c_void_p()
    _native.check(lib.pb_env_create(C.byref(cfg), C.byref(h)))
    info = _native.EnvInfo()
    _native.check(lib.pb_env_get_info(h, C.byref(info)))
    assert info.obs_dtype == _native.DTYPE_U8 and info.obs_bytes == ROW and info.num_actions == 4
    assert tuple(info.obs_shape[:3]) == SHAPE and info.obs_low == 0 and info.obs_high == 255
    obs = torch.zeros(n * (ROW + 32) + 16, dtype=torch.uint8, device='cuda')
    rew = torch.zeros(n, device='cuda')
    flags = torch.zeros(3, n, dtype=torch.uint8, device='cuda')
    dones = torch.zeros(n, device='cuda')
    acts = torch.zeros(n, dtype=torch.int64, device='cuda')

    def out(offset, stride):
        return _native.EnvOut(obs=obs.data_ptr() + offset, obs_stride=stride, rewards=rew.data_ptr(),
                              terminals=flags[0].data_ptr(), truncations=flags[1].data_ptr(), masks=flags[2].data_ptr(),
                              dones_f32=dones.data_ptr())
    s = _native.stream_ptr()
    for offset, stride in ((1, ROW), (0, ROW + 8)):
        l0 = lib.pb_launch_count()
        assert lib.pb_env_reset(h, C.c_uint64(1), C.byref(out(offset, stride)), s) == _native.PB_ERR_INVALID
        assert lib.pb_launch_count() == l0, (offset, stride)
    _native.check(lib.pb_env_reset(h, C.c_uint64(1), C.byref(out(0, ROW)), s))
    for offset, stride in ((8, ROW), (0, ROW + 4)):
        l0 = lib.pb_launch_count()
        assert lib.pb_env_step(h, C.c_void_p(acts.data_ptr()), C.byref(out(offset, stride)), s) == _native.PB_ERR_INVALID
        assert lib.pb_launch_count() == l0, (offset, stride)
    torch.cuda.synchronize()
    lib.pb_env_destroy(h)


# ---- 4. training: models.Convolutional through create / evaluate / train ---------------------------------------------
def test_convolutional_trains_captured(monkeypatch):
    """Convolutional(framestack=4, flat_size=3136) behind cleanrl.Policy at 256 envs x 32 steps, cuda_graph=True, three
    evaluate() + train() iterations: every stored row replays bit-exactly through the oracle, conv1 runs on the uint8
    fast path (_Conv1U8Function), the rollout and the update are captured graphs, losses are finite, parameters move."""
    n, h = 256, 32
    calls = []
    orig = models._Conv1U8Function.apply
    monkeypatch.setattr(models._Conv1U8Function, 'apply', lambda *a: calls.append(1) or orig(*a))
    vec = pvec.make(ocean.env_creator(KIND), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Convolutional(vec.driver_env, framestack=4, flat_size=3136), fused_sample=True,
                         seed=3).cuda()
    cfg = pufferlib_b200.namespace(
        seed=1, torch_deterministic=True, env=KIND, batch_size=n * h, bptt_horizon=8, minibatch_size=n * h // 2,
        cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
        update_epochs=1, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01,
        max_grad_norm=0.5, target_kl=None, anneal_lr=False, total_timesteps=10 ** 9, cuda_graph=True)
    data = clean_pufferl.create(cfg, vec, pol)
    ora = oracle(n)
    ora.collect_infos = False
    ora.async_reset(1)
    for it in range(3):
        clean_pufferl.evaluate(data)
        exp = data.experience
        acts, obs = cpu(exp.actions).reshape(h, n), cpu(exp.obs).reshape(h, n, *SHAPE)
        rew, done = cpu(exp.rewards).reshape(h, n), cpu(exp.dones).reshape(h, n)
        for t in range(h):
            o, r, d, _, _, _, _ = ora.recv()
            assert np.array_equal(o, obs[t]), (it, t)
            assert np.array_equal(r, rew[t]) and np.array_equal(d.astype(np.float32), done[t]), (it, t)
            ora.send(acts[t])
        before = [p.detach().clone() for p in pol.parameters()]
        clean_pufferl.train(data)
        losses = [data.losses.policy_loss, data.losses.value_loss, data.losses.entropy]
        assert all(np.isfinite(x) for x in losses), (it, losses)
        moved = [not torch.equal(a, p.detach()) for a, p in zip(before, pol.parameters())]
        assert all(moved), (it, moved)
    assert data.graph_state == 2 and data.train_graph_state == 2, (data.graph_state, data.train_graph_state)
    assert data.graph_replays >= 1
    assert calls, 'conv1 must run on the uint8 fast path (the captured graphs hold the calls made while capturing)'
    clean_pufferl.close(data)
    ora.close()
