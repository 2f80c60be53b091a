"""Device ocean test envs (memory, password, stochastic, bandit) + vectoriser vs the reference's own trajectories
(tests/golden/ocean_*.npz) and vs the oracle at scale: bitwise obs, reward bits, terminals, truncations, masks;
EpisodeStats infos to 1e-12; the device statistics reduction."""
import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from oracle.ocean import OceanSerial
from pufferlib_b200.environments import ocean
from pufferlib_b200.exceptions import APIUsageError
from test_ocean_cpu import MP_CASES, SERIAL_CASES, golden_kwargs

pytestmark = pytest.mark.gpu


def to_np(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def check_infos(got, ref):
    got = np.asarray(got, dtype=np.float64).reshape(-1, 5)
    assert got.shape == ref.shape
    assert np.array_equal(got[:, [0, 1, 3]], ref[:, [0, 1, 3]])
    assert np.allclose(got[:, [2, 4]], ref[:, [2, 4]], rtol=1e-12, atol=1e-15)   # fp64 sums vs python's sum


def make_vec(g, backend, **kw):
    n = int(g['num_envs'])
    w = int(g['num_workers'])
    if w:
        kw.update(num_workers=w, batch_size=n)
    return pvec.make(ocean.env_creator(str(g['kind'])), env_kwargs=golden_kwargs(g), num_envs=n, backend=backend, **kw)


def run_case(g, backend, actions_on_device, bound=False):
    n, seed, h = int(g['num_envs']), int(g['seed']), int(g['horizon'])
    vec = make_vec(g, backend)
    if int(g['num_workers']):
        assert len(vec._shards) == int(g['num_workers'])
    if bound:
        from pufferlib_b200 import clean_pufferl
        exp = clean_pufferl.Experience(n * 8, 4, n * 8, g['obs'].shape[2:], np.float32, ())
        vec.bind_rollout(exp)
    vec.async_reset(seed)
    info_rows = []
    for t in range(h + 1):
        o, r, term, trunc, infos, ids, mask = vec.recv()
        assert np.array_equal(to_np(o).view(np.uint32), g['obs'][t].view(np.uint32)), f'obs step {t}'
        assert np.array_equal(to_np(r).view(np.uint32), g['rewards'][t].view(np.uint32)), f'reward bits step {t}'
        assert np.array_equal(to_np(term), g['terminals'][t]), f'terminals step {t}'
        assert np.array_equal(to_np(trunc), g['truncations'][t])
        assert np.array_equal(to_np(mask), g['masks'][t])
        assert np.array_equal(ids, np.arange(n))
        for k, i in enumerate(infos):
            info_rows.append((t, k, i['episode_return'], i['episode_length'], i['score']))
        if t < h:
            a = g['actions'][t]
            if bound:
                a = torch.as_tensor(a, device='cuda')
                z = torch.zeros(n, device='cuda')
                exp.store(o, z, a, z, r, term, ids, mask)
                if exp.full:
                    exp.sort_training_data()
            vec.send(torch.as_tensor(a, device='cuda') if actions_on_device else a)
    check_infos(info_rows, g['infos'])
    vec.close()


@pytest.mark.parametrize('case', SERIAL_CASES + MP_CASES)
def test_ocean_device_tensors(golden, case):
    run_case(golden(case), pvec.B200.options(exact_infos=True), actions_on_device=True)


@pytest.mark.parametrize('case', SERIAL_CASES + MP_CASES)
def test_ocean_host_buffers(golden, case):
    """host_buffers=True: numpy in / numpy out like vector.Serial."""
    run_case(golden(case), pvec.B200.options(host_buffers=True), actions_on_device=False)


@pytest.mark.parametrize('case', SERIAL_CASES + MP_CASES)
def test_ocean_bound_rollout(golden, case):
    """send() writing obs / reward / done rows straight into a bound Experience."""
    run_case(golden(case), pvec.B200.options(exact_infos=True), actions_on_device=True, bound=True)


@pytest.mark.parametrize('case', SERIAL_CASES)
def test_ocean_episode_stats(golden, case):
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
    assert count == len(ref)
    for k, col in (('episode_return', 2), ('episode_length', 3), ('score', 4)):
        assert np.isclose(means[k], ref[:, col].mean(), rtol=1e-9, atol=1e-12), k
    vec.close()


def test_memory_pool_mode_matches_multiprocessing(golden):
    """Pool mode (batch_size = one worker's envs): groups come back round-robin, every env follows the reference
    Multiprocessing trajectory (one np.random stream per worker)."""
    g = golden('ocean_memory_mp_n12_w4')
    n, w, seed, h = int(g['num_envs']), int(g['num_workers']), int(g['seed']), int(g['horizon'])
    b = n // w
    vec = pvec.make(ocean.env_creator('memory'), num_envs=n, num_workers=w, batch_size=b, backend=pvec.B200)
    assert isinstance(vec, pvec.B200Pool) and len(vec.groups) == w
    vec.async_reset(seed)
    for t in range(h + 1):
        for k in range(w):
            o, r, d, tr, infos, ids, m = vec.recv()
            lo, hi = k * b, (k + 1) * b
            assert np.array_equal(ids, np.arange(lo, hi))
            assert np.array_equal(to_np(o), g['obs'][t, lo:hi]), (t, k)
            assert np.array_equal(to_np(r).view(np.uint32), g['rewards'][t, lo:hi].view(np.uint32)), (t, k)
            assert np.array_equal(to_np(d), g['terminals'][t, lo:hi])
            vec.send(torch.as_tensor(g['actions'][min(t, h - 1), lo:hi], device='cuda'))
    vec.close()


@pytest.mark.parametrize('kind,kwargs,steps', [('memory', {}, 24), ('memory', {'mem_length': 5, 'mem_delay': 3}, 30),
                                               ('password', {}, 14), ('stochastic', {'p': 0.3}, 210),
                                               ('bandit', {}, 6), ('bandit', {'num_actions': 7, 'reward_scale': 0.5}, 6)])
def test_ocean_matches_oracle_at_scale(kind, kwargs, steps):
    """N = 16 384 against the oracle: many twists of the memory stream per reset-send, ragged last warp in none,
    the bandit's 16 384 gaussians (device log vs libm log)."""
    n, seed = 16384, 1000
    n_act = kwargs.get('num_actions', 10) if kind == 'bandit' else 2
    rng = np.random.default_rng(5)
    vec = pvec.make(ocean.env_creator(kind), env_kwargs=kwargs, num_envs=n, backend=pvec.B200.options(exact_infos=True))
    ora = OceanSerial(kind, n, **kwargs)
    vec.async_reset(seed)
    ora.async_reset(seed)
    for t in range(steps + 1):
        o, r, term, trunc, infos, ids, mask = vec.recv()
        oo, orr, ot, otr, oinf, _, om = ora.recv()
        assert np.array_equal(to_np(o), oo), t
        assert np.array_equal(to_np(r).view(np.uint32), orr.view(np.uint32)), t
        assert np.array_equal(to_np(term), ot), t
        assert len(infos) == len(oinf)
        if infos:
            got = np.asarray([[i['episode_return'], i['episode_length'], i['score']] for i in infos])
            ref = np.asarray([[i['episode_return'], i['episode_length'], i['score']] for i in oinf])
            assert np.allclose(got, ref, rtol=1e-12, atol=1e-15), t
        if t < steps:
            a = rng.integers(0, n_act, size=n)
            vec.send(a)
            ora.send(a)
    vec.close()


def test_memory_seeds():
    """Seed lists, seeds np.random.seed refuses, and shards seeded by global env index."""
    n = 6
    ref = OceanSerial('memory', n)
    ref.async_reset(100)
    vec = pvec.make(ocean.env_creator('memory'), num_envs=n, backend=pvec.B200)
    vec.async_reset([100 + i for i in range(n)])
    assert np.array_equal(to_np(vec.recv()[0]), ref.observations)
    with pytest.raises(APIUsageError):
        vec.async_reset(2 ** 32 - n + 1)            # seed + N - 1 >= 2**32
    vec.async_reset(2 ** 32 - n)                   # the largest accepted
    vec.recv()
    with pytest.raises(APIUsageError):
        vec.async_reset(-1)
    vec.close()
    with pytest.raises(APIUsageError):            # stochastic seeds np.random too
        s = pvec.make(ocean.env_creator('stochastic'), num_envs=2, backend=pvec.B200)
        s.async_reset(2 ** 32)
    # bandit and password reseed 42 whatever the seed
    b = pvec.make(ocean.env_creator('bandit'), num_envs=2, backend=pvec.B200)
    b.async_reset(2 ** 40)
    b.close()
    # env_index_offset: a shard seeds env i with seed + offset + i
    off = pvec.make(ocean.env_creator('memory'), num_envs=3, backend=pvec.B200.options(env_index_offset=3))
    off.async_reset(100)
    assert np.array_equal(to_np(off.recv()[0]), ref.observations[3:])
    off.close()


def test_out_of_envelope_refused_by_the_library():
    """pb_env_create_ex itself refuses out-of-envelope parameters (the host layer refuses them before)."""
    import ctypes as C
    from pufferlib_b200 import _native
    lib = _native.lib()
    for kind, ip, dp in (('memory', [65, 0], []), ('memory', [2, 1026], []), ('password', [129], []),
                         ('bandit', [40000], []), ('bandit', [4], [float('nan'), 1.0]), ('stochastic', [], [float('inf')])):
        cfg = _native.EnvConfig(kind=_native.ENV_KINDS[kind], num_envs=4, device=0,
                                iparam=(C.c_int32 * 8)(*(ip + [0] * (8 - len(ip)))))
        h = C.c_void_p()
        arr = (C.c_double * max(len(dp), 1))(*dp)
        assert lib.pb_env_create_ex(C.byref(cfg), arr, len(dp), C.byref(h)) == _native.PB_ERR_INVALID, (kind, ip, dp)
        assert not h.value


def test_spaces_from_the_library():
    for kind, kw, shape, lo, hi, n_act in (('memory', {}, (1,), -1, 1, 2), ('password', {'password_length': 9}, (9,), 0, 1, 2),
                                           ('stochastic', {}, (1,), 0, 1, 2), ('bandit', {'num_actions': 3}, (1,), -1, 1, 3)):
        vec = pvec.make(ocean.env_creator(kind), env_kwargs=kw, num_envs=2, backend=pvec.B200)
        sp = vec.single_observation_space
        assert sp.shape == shape and sp.dtype == np.float32 and float(sp.low.min()) == lo and float(sp.high.max()) == hi
        assert vec.single_action_space.n == n_act
        vec.close()


@pytest.mark.parametrize('case', ['squared_c1', 'squared_d2_n33', 'squared_mp_n12_w4'])
def test_squared_golden_after_mt_header(golden, case):
    """Squared's MT19937 pieces now come from mt19937.cuh, shared with memory: its outputs are unchanged."""
    g = golden(case)
    n, seed, h = int(g['num_envs']), int(g['seed']), int(g['horizon'])
    w = int(g['num_workers']) if 'num_workers' in g else 0
    kw = dict(num_workers=w, batch_size=n) if w else {}
    d = int(g['distance_to_target']) if 'distance_to_target' in g else 3
    vec = pvec.make(ocean.env_creator('squared'), env_kwargs={'distance_to_target': d}, num_envs=n,
                    backend=pvec.B200.options(exact_infos=True), **kw)
    vec.async_reset(seed)
    for t in range(h + 1):
        o, r, term, trunc, infos, ids, mask = vec.recv()
        assert np.array_equal(to_np(o), g['obs_i8'][t].astype(np.float32)), t
        assert np.array_equal(to_np(r).view(np.uint32), g['rewards'][t].view(np.uint32)), t
        if t < h:
            vec.send(torch.as_tensor(g['actions'][t], device='cuda'))
    vec.close()
