"""The ocean test envs (memory, password, stochastic, bandit) without a device: how creators resolve to native kinds,
which parameters are refused, and the oracle (oracle/ocean.py) against the reference's own trajectories
(tests/golden/ocean_*.npz): bitwise rows, infos to 1e-12."""
import numpy as np
import pytest

from oracle.ocean import NumpyLegacyRandom, OceanMultiprocessing, OceanSerial
from pufferlib_b200.environments import GLOBAL_STREAM_KINDS, ocean, resolve, resolve_config
from pufferlib_b200.exceptions import APIUsageError

SERIAL_CASES = ['ocean_memory_n5', 'ocean_memory_n1', 'ocean_memory_l3d5_n33', 'ocean_password_n5',
                'ocean_password_l7_n33', 'ocean_stochastic_n3', 'ocean_stochastic_p025_n33', 'ocean_bandit_n5',
                'ocean_bandit_n1', 'ocean_bandit_a4_noise0_n33', 'ocean_bandit_a4_noise1_n33']
MP_CASES = ['ocean_memory_mp_n12_w4', 'ocean_bandit_mp_n8_w2']


def golden_kwargs(g):
    kw = {}
    for k, v in zip(g['env_kwargs_keys'], g['env_kwargs_values']):
        kw[str(k)] = float(v) if str(k) in ('p', 'reward_scale', 'reward_noise') else int(v)
    return kw


def test_resolve_defaults_args_and_kwargs():
    c = ocean.env_creator
    assert resolve_config(c('memory'), [], {}) == ('memory', [2, 3, 0, 0, 0, 0, 0, 0], [])
    assert resolve(c('memory'), [3, 5], {}) == ('memory', [3, 6, 0, 0, 0, 0, 0, 0])
    assert resolve(c('memory'), [4], {'mem_delay': 0})[1][:2] == [4, 1]
    assert resolve_config(c('password'), [], {}) == ('password', [5] + [0] * 7, [])
    assert resolve(c('password'), [], {'password_length': 7})[1][0] == 7
    assert resolve_config(c('stochastic'), [], {}) == ('stochastic', [0] * 8, [0.7])
    assert resolve_config(c('stochastic'), [0.25, 1000], {})[2] == [0.25]          # horizon accepted and ignored
    assert resolve_config(c('stochastic'), [], {'p': 0.5, 'horizon': 7})[2] == [0.5]
    assert resolve_config(c('bandit'), [], {}) == ('bandit', [10] + [0] * 7, [1.0, 1.0])
    assert resolve_config(c('bandit'), [4], {'reward_noise': 0}) == ('bandit', [4] + [0] * 7, [1.0, 0.0])
    assert resolve_config(c('bandit'), [4, 2.5, 0.5], {})[2] == [2.5, 0.5]

    def make_memory(mem_length=2, mem_delay=2):     # the reference's creators are recognised by name
        pass

    def make_bandit():
        pass
    assert resolve(make_memory, [], {})[0] == 'memory'
    assert resolve(make_bandit, [], {'num_actions': 3})[1][0] == 3
    for name in ('memory', 'password', 'stochastic', 'bandit'):
        assert ocean.env_creator(name).__name__ == 'make_' + name
        with pytest.raises(APIUsageError):
            ocean.env_creator(name)()                # no CPU instantiation
    assert GLOBAL_STREAM_KINDS == {'squared', 'memory', 'bandit'}


@pytest.mark.parametrize('kind,args,kwargs', [
    ('memory', [0], {}), ('memory', [65], {}), ('memory', [], {'mem_delay': -1}), ('memory', [], {'mem_delay': 1025}),
    ('memory', [2.5], {}), ('memory', [], {'bogus': 1}), ('memory', [1, 2, 3], {}),
    ('password', [0], {}), ('password', [129], {}), ('password', [], {'length': 5}),
    ('stochastic', [float('nan')], {}), ('stochastic', [], {'q': 0.5}),
    ('bandit', [0], {}), ('bandit', [2 ** 15 + 1], {}), ('bandit', [4, float('inf')], {}), ('bandit', [], {'x': 1}),
])
def test_resolve_refusals(kind, args, kwargs):
    with pytest.raises(APIUsageError):
        resolve(ocean.env_creator(kind), args, kwargs)


def test_numpy_legacy_random_matches_numpy():
    rs = np.random.RandomState()
    ours = NumpyLegacyRandom()
    for seed in (0, 42, 7, 2 ** 32 - 1):
        rs.seed(seed)
        ours.seed(seed)
        assert [int(rs.randint(0, 10)) for _ in range(50)] == [ours.randint(10) for _ in range(50)]
        assert list(rs.randint(0, 2, size=700)) == [ours.randint(2) for _ in range(700)]
        assert [rs.randn() for _ in range(301)] == [ours.randn() for _ in range(301)]
        assert [int(rs.randint(0, 1)) for _ in range(3)] == [ours.randint(1) for _ in range(3)]
    with pytest.raises(ValueError):
        ours.seed(2 ** 32)
    with pytest.raises(ValueError):
        ours.seed(-1)


def run_oracle(vec, g):
    h = int(g['horizon'])
    rows, infos = [], []
    for t in range(h + 1):
        o, r, d, tr, info, ids, m = vec.recv()
        rows.append((o.copy(), r.copy(), d.copy(), tr.copy(), m.copy()))
        for k, i in enumerate(info):
            infos.append((t, k, i['episode_return'], i['episode_length'], i['score']))
        if t < h:
            vec.send(g['actions'][t])
    return rows, np.asarray(infos, dtype=np.float64).reshape(-1, 5)


def check_rows(rows, infos, g):
    for t, (o, r, d, tr, m) in enumerate(rows):
        assert np.array_equal(o.view(np.uint32), g['obs'][t].view(np.uint32)), f'obs step {t}'
        assert np.array_equal(r.view(np.uint32), g['rewards'][t].view(np.uint32)), f'reward bits step {t}'
        assert np.array_equal(d, g['terminals'][t]) and np.array_equal(tr, g['truncations'][t])
        assert np.array_equal(m, g['masks'][t])
    ref = g['infos']
    assert infos.shape == ref.shape
    assert np.array_equal(infos[:, [0, 1, 3]], ref[:, [0, 1, 3]])
    assert np.allclose(infos[:, [2, 4]], ref[:, [2, 4]], rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize('case', SERIAL_CASES)
def test_ocean_oracle_vs_reference_serial(golden, case):
    g = golden(case)
    vec = OceanSerial(str(g['kind']), int(g['num_envs']), **golden_kwargs(g))
    vec.async_reset(int(g['seed']))
    check_rows(*run_oracle(vec, g), g)


@pytest.mark.parametrize('case', MP_CASES)
def test_ocean_oracle_vs_reference_multiprocessing(golden, case):
    g = golden(case)
    vec = OceanMultiprocessing(str(g['kind']), int(g['num_envs']), int(g['num_workers']), **golden_kwargs(g))
    vec.async_reset(int(g['seed']))
    check_rows(*run_oracle(vec, g), g)


def test_goldens_cover_what_they_are_for(golden):
    """Each golden runs long enough for several episodes per env, and the bandit noise really is shared per env."""
    for case in SERIAL_CASES + MP_CASES:
        g = golden(case)
        assert g['terminals'].sum(axis=0).min() >= 3, case
    g = golden('ocean_bandit_n5')
    steps = [t for t in range(1, int(g['horizon']) + 1) if g['terminals'][t].all()]
    noise = [g['rewards'][t].astype(np.float64) - (g['actions'][t - 1] == 6) for t in steps]   # arm 6 wins at 10 arms
    assert len(steps) >= 3 and all(np.allclose(noise[0], x, rtol=0, atol=1e-6) for x in noise)
    assert np.ptp(noise[0]) > 0.1
