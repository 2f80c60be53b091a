"""The multiagent ocean env without a device: how its creator resolves (it takes no arguments), and the oracle
(tests/multiagent_oracle.py) against the reference's own trajectories (tests/golden/multiagent_*.npz), bitwise,
infos included."""
import numpy as np
import pytest

from multiagent_oracle import MultiagentMultiprocessing, MultiagentSerial, info_rows
from pufferlib_b200.environments import GLOBAL_STREAM_KINDS, ocean, resolve_config
from pufferlib_b200.exceptions import APIUsageError

SERIAL_CASES = ['multiagent_n1', 'multiagent_n5', 'multiagent_n33']
MP_CASES = ['multiagent_mp_n8_w2']


def test_resolve_takes_no_arguments():
    c = ocean.env_creator('multiagent')
    assert c.__name__ == 'make_multiagent'
    assert resolve_config(c, [], {}) == ('multiagent', [0] * 8, [])
    assert resolve_config(c, None, None) == ('multiagent', [0] * 8, [])

    def make_multiagent():                 # the reference's creator is recognised by name
        pass
    assert resolve_config(make_multiagent, [], {})[0] == 'multiagent'
    for args, kwargs in (([1], {}), ([], {'num_agents': 2}), ([0], {}), ([], {'seed': 1})):
        with pytest.raises(APIUsageError):
            resolve_config(c, args, kwargs)
    with pytest.raises(APIUsageError):
        c()                                # no CPU instantiation
    assert 'multiagent' not in GLOBAL_STREAM_KINDS


def run_oracle(vec, g):
    h = int(g['horizon'])
    rows, infos = [], []
    for t in range(h + 1):
        o, r, d, tr, info, ids, m = vec.recv()
        assert np.array_equal(ids, np.arange(2 * int(g['num_envs'])))
        rows.append((o.copy(), r.copy(), d.copy(), tr.copy(), m.copy()))
        for i in info:
            assert sorted(i) == [1, 2] and all(type(i[a]['score']) is int for a in (1, 2))
        infos += info_rows(t, info)
        if t < h:
            vec.send(g['actions'][t])
    return rows, np.asarray(infos, dtype=np.int64).reshape(-1, 4)


def check_rows(rows, infos, g):
    for t, (o, r, d, tr, m) in enumerate(rows):
        assert np.array_equal(o.view(np.uint32), g['obs'][t].view(np.uint32)), f'obs step {t}'
        assert np.array_equal(r.view(np.uint32), g['rewards'][t].view(np.uint32)), f'reward bits step {t}'
        assert np.array_equal(d, g['terminals'][t]) and np.array_equal(tr, g['truncations'][t])
        assert np.array_equal(m, g['masks'][t])
    assert np.array_equal(infos, g['infos'])


@pytest.mark.parametrize('case', SERIAL_CASES)
def test_multiagent_oracle_vs_reference_serial(golden, case):
    g = golden(case)
    vec = MultiagentSerial(int(g['num_envs']))
    vec.async_reset(int(g['seed']))
    check_rows(*run_oracle(vec, g), g)


@pytest.mark.parametrize('case', MP_CASES)
def test_multiagent_oracle_vs_reference_multiprocessing(golden, case):
    g = golden(case)
    vec = MultiagentMultiprocessing(int(g['num_envs']), int(g['num_workers']))
    vec.async_reset(int(g['seed']))
    check_rows(*run_oracle(vec, g), g)


def test_goldens_cover_what_they_are_for(golden):
    """Rows are agent-major within an env, every second send is a reset-send, and both rewards occur for both agents."""
    for case in SERIAL_CASES + MP_CASES:
        g = golden(case)
        n, h = int(g['num_envs']), int(g['horizon'])
        assert h >= 6 and g['obs'].shape == (h + 1, 2 * n, 1)
        assert np.array_equal(g['obs'][:, 0::2], np.zeros((h + 1, n, 1), np.float32))
        assert np.array_equal(g['obs'][:, 1::2], np.ones((h + 1, n, 1), np.float32))
        assert g['terminals'][0::2].sum() == 0 and g['terminals'][1::2].all()
        assert len(g['infos']) == 2 * n * ((h + 1) // 2)
        if n >= 5:
            for agent in (1, 2):
                assert set(g['infos'][g['infos'][:, 2] == agent, 3]) == {0, 1}
