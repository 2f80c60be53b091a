"""Generate the multiagent golden vectors by running the UNMODIFIED reference (a PufferLib source checkout named by
PUFFERLIB_REFERENCE).

    PUFFERLIB_REFERENCE=<checkout> python tests/golden/generate_multiagent.py   # writes tests/golden/multiagent_*.npz

multiagent_*.npz   pufferlib.vector.make(ocean.env_creator('multiagent'), backend=Serial) -- and Multiprocessing with
                   batch_size == num_envs -- driven by a fixed action tape over the 2 * num_envs agent rows
                   (np.random.default_rng); every recv() row (float32 obs / reward / terminal / trunc / mask) and every
                   info dict as (recv index, dict index, agent, score) rows.
                                                  [ocean.py:149-208, emulation.py:236-420, vector.py:70-190, 345-401]

Like generate_ocean.py this runs the reference on the stand-ins of ``oracle/shim`` (gymnasium / gym / pettingzoo are not
installed).  The reference's Serial.close() calls each env's close(), which PettingZooPufferEnv forwards to the
pettingzoo ParallelEnv base class: real pettingzoo's is a no-op, so the same no-op is given to the stand-in here.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(REPO, 'oracle', 'shim'), os.environ['PUFFERLIB_REFERENCE']]

import warnings
warnings.filterwarnings('ignore')
import numpy as np
import pettingzoo

import pufferlib
import pufferlib.vector
from pufferlib.environments import ocean

if not hasattr(pettingzoo.ParallelEnv, 'close'):
    pettingzoo.ParallelEnv.close = lambda self: None


def action_tape(horizon, rows, seed):
    return np.random.default_rng(seed).integers(0, 2, size=(horizon, rows), dtype=np.int64)


def run_multiagent(num_envs, seed, horizon, num_workers=None):
    """An action tape through the reference's Serial (or synchronous Multiprocessing) over the multiagent env; every
    recv() row and info dict.  The info values must be python ints keyed by the agents 1 and 2."""
    if num_workers:
        vec = pufferlib.vector.make(ocean.env_creator('multiagent'), num_envs=num_envs, num_workers=num_workers,
                                    batch_size=num_envs, backend=pufferlib.vector.Multiprocessing)
    else:
        vec = pufferlib.vector.make(ocean.env_creator('multiagent'), num_envs=num_envs,
                                    backend=pufferlib.vector.Serial)
    rows = 2 * num_envs
    assert vec.num_agents == rows and vec.agents_per_batch == rows
    tape = action_tape(horizon, rows, seed=seed % 1000)
    obs, rew, term, trunc, mask, info_rows = [], [], [], [], [], []
    vec.async_reset(seed)
    for t in range(horizon + 1):
        o, r, d, tr, infos, env_id, m = vec.recv()
        assert np.array_equal(np.asarray(env_id).ravel(), np.arange(rows))
        obs.append(np.asarray(o).reshape(rows, -1).copy()); rew.append(np.asarray(r).reshape(rows).copy())
        term.append(np.asarray(d).reshape(rows).copy()); trunc.append(np.asarray(tr).reshape(rows).copy())
        mask.append(np.asarray(m).reshape(rows).copy())
        for k, i in enumerate(infos):
            assert sorted(i) == [1, 2], i
            for agent in (1, 2):
                assert sorted(i[agent]) == ['score'] and type(i[agent]['score']) is int, i
                info_rows.append((t, k, agent, i[agent]['score']))
        if t < horizon:
            vec.send(tape[t])
    vec.close()
    return dict(kind='multiagent', num_envs=num_envs, seed=seed, horizon=horizon, actions=tape,
                num_workers=num_workers or 0, obs=np.stack(obs), rewards=np.stack(rew), terminals=np.stack(term),
                truncations=np.stack(trunc), masks=np.stack(mask),
                infos=np.asarray(info_rows, dtype=np.int64).reshape(-1, 4))


MULTIAGENT_CASES = {
    'multiagent_n1': dict(num_envs=1, seed=42, horizon=8),
    'multiagent_n5': dict(num_envs=5, seed=7, horizon=12),
    'multiagent_n33': dict(num_envs=33, seed=123456, horizon=15),
    'multiagent_mp_n8_w2': dict(num_envs=8, seed=3, horizon=10, num_workers=2),
}


def gen_multiagent():
    for name, kw in MULTIAGENT_CASES.items():
        out = run_multiagent(**kw)
        np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
        print(name, out['obs'].shape, 'infos', out['infos'].shape)


if __name__ == '__main__':
    gen_multiagent()
