"""Generate the ocean test-env golden vectors by running the UNMODIFIED reference (a PufferLib source checkout named by
PUFFERLIB_REFERENCE).

    PUFFERLIB_REFERENCE=<checkout> python tests/golden/generate_ocean.py      # writes tests/golden/ocean_*.npz

ocean_*.npz   pufferlib.vector.make(ocean.env_creator(kind), backend=Serial) -- and Multiprocessing with
              batch_size == num_envs -- over memory / password / stochastic / bandit, driven by a fixed action tape
              (np.random.default_rng); every recv() row (float32 obs / reward / terminal / trunc / mask) and every info
              dict.                                       [ocean.py:8-123, 228-281, 529-582, vector.py:70-190, 345-401]

The tests must not need the reference, so its outputs are committed next to this file as small fixtures.  gymnasium /
gym / pettingzoo are not installed in this image; ``oracle/shim`` provides stand-ins for the handful of classes the
reference touches on this path (the reference source itself is not modified).  generate.py makes the other goldens.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(REPO, 'oracle', 'shim'), os.environ['PUFFERLIB_REFERENCE']]

import warnings
warnings.filterwarnings('ignore')
import numpy as np

import pufferlib
import pufferlib.vector
from pufferlib.environments import ocean


def action_tape(horizon, num_envs, n_act, seed):
    return np.random.default_rng(seed).integers(0, n_act, size=(horizon, num_envs), dtype=np.int64)


OCEAN_N_ACT = {'memory': 2, 'password': 2, 'stochastic': 2}


def run_ocean(kind, num_envs, seed, horizon, env_kwargs=None, num_workers=None):
    """An action tape through the reference's Serial (or synchronous Multiprocessing) over one ocean env kind; every
    recv() row and info dict.  Password's reset observation (-1) lies outside its own Box(0, 1): the emulation layer's
    one-time check_space (emulation.py:183-185) would refuse it, so the Serial envs are marked as checked first;
    nothing else is touched."""
    env_kwargs = env_kwargs or {}
    n_act = OCEAN_N_ACT.get(kind) or env_kwargs.get('num_actions', 10)
    if num_workers:
        vec = pufferlib.vector.make(ocean.env_creator(kind), env_kwargs=env_kwargs, num_envs=num_envs,
                                    num_workers=num_workers, batch_size=num_envs,
                                    backend=pufferlib.vector.Multiprocessing)
    else:
        vec = pufferlib.vector.make(ocean.env_creator(kind), env_kwargs=env_kwargs, num_envs=num_envs,
                                    backend=pufferlib.vector.Serial)
        if kind == 'password':
            for e in vec.envs:
                e.is_observation_checked = True
    tape = action_tape(horizon, num_envs, n_act=n_act, seed=seed % 1000)
    obs, rew, term, trunc, mask, info_rows = [], [], [], [], [], []
    vec.async_reset(seed)
    for t in range(horizon + 1):
        o, r, d, tr, infos, env_id, m = vec.recv()
        assert np.array_equal(env_id, np.arange(num_envs))
        obs.append(o.copy()); rew.append(r.copy()); term.append(d.copy()); trunc.append(tr.copy()); mask.append(m.copy())
        for k, i in enumerate(infos):
            info_rows.append((t, k, i['episode_return'], i['episode_length'], float(i['score'])))
        if t < horizon:
            vec.send(tape[t])
    vec.close()
    return dict(kind=kind, num_envs=num_envs, seed=seed, horizon=horizon, actions=tape,
                env_kwargs_keys=np.asarray(sorted(env_kwargs), dtype=str),
                env_kwargs_values=np.asarray([float(env_kwargs[k]) for k in sorted(env_kwargs)], dtype=np.float64),
                num_workers=num_workers or 0, obs=np.stack(obs), rewards=np.stack(rew), terminals=np.stack(term),
                truncations=np.stack(trunc), masks=np.stack(mask),
                infos=np.asarray(info_rows, dtype=np.float64).reshape(-1, 5))


OCEAN_CASES = {
    'ocean_memory_n5': dict(kind='memory', num_envs=5, seed=42, horizon=30),
    'ocean_memory_n1': dict(kind='memory', num_envs=1, seed=7, horizon=20),
    'ocean_memory_l3d5_n33': dict(kind='memory', num_envs=33, seed=123456, horizon=60,
                                  env_kwargs={'mem_length': 3, 'mem_delay': 5}),
    'ocean_password_n5': dict(kind='password', num_envs=5, seed=1, horizon=24),
    'ocean_password_l7_n33': dict(kind='password', num_envs=33, seed=3, horizon=30, env_kwargs={'password_length': 7}),
    'ocean_stochastic_n3': dict(kind='stochastic', num_envs=3, seed=5, horizon=310),
    'ocean_stochastic_p025_n33': dict(kind='stochastic', num_envs=33, seed=2**31 + 9, horizon=310,
                                      env_kwargs={'p': 0.25}),
    'ocean_bandit_n5': dict(kind='bandit', num_envs=5, seed=42, horizon=12),
    'ocean_bandit_n1': dict(kind='bandit', num_envs=1, seed=0, horizon=9),
    'ocean_bandit_a4_noise0_n33': dict(kind='bandit', num_envs=33, seed=11, horizon=10,
                                       env_kwargs={'num_actions': 4, 'reward_noise': 0}),
    'ocean_bandit_a4_noise1_n33': dict(kind='bandit', num_envs=33, seed=11, horizon=10,
                                       env_kwargs={'num_actions': 4, 'reward_noise': 1}),
    'ocean_memory_mp_n12_w4': dict(kind='memory', num_envs=12, seed=5, horizon=30, num_workers=4),
    'ocean_bandit_mp_n8_w2': dict(kind='bandit', num_envs=8, seed=3, horizon=8, num_workers=2),
}


def gen_ocean():
    for name, kw in OCEAN_CASES.items():
        out = run_ocean(**kw)
        np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
        print(name, out['obs'].shape, 'infos', out['infos'].shape)


if __name__ == '__main__':
    gen_ocean()
