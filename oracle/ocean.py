"""``vector.Serial`` / ``vector.Multiprocessing`` over the reference's ocean test envs Memory, Password, Stochastic
and Bandit, restated over numpy arrays.  TEST INFRASTRUCTURE.

Follows (all under reference pufferlib/):
  environments/ocean/ocean.py:8-62       Bandit      (reseeds 42 on every reset; one-step episodes)
  environments/ocean/ocean.py:64-123     Memory      (np.random.randint(0, 2, size=2L+D) per reset)
  environments/ocean/ocean.py:228-281    Password    (reseeds 42 on every reset; obs starts at -1)
  environments/ocean/ocean.py:529-582    Stochastic  (no RNG; python-double reward)
  environments/ocean/environment.py:33-46, 67-70   creator defaults (make_stochastic passes horizon=100)
  postprocess.py:8-54                    EpisodeStats (builtin sum of the per-step values on the done row)
  emulation.py:169-228                   buffer rows: reset -> r=0, term=False, trunc=False, mask=True
  vector.py:112-162, 639-641             Serial: seeds seed+i; `if env.done: reset() else: step()` per send

RNG: numpy's legacy process-global ``np.random`` restated on oracle/mt19937.py: ``np.random.seed(int)`` is
``init_genrand`` (and refuses seeds outside [0, 2**32)), ``randint(0, n)`` is masked rejection on 32-bit outputs,
``randn()`` is the legacy polar method with the second value of each pair cached.  Every env of a Serial shares the
one stream, in env order; every Multiprocessing worker has its own.
"""
import math

import numpy as np

from .mt19937 import MT19937

DEFAULTS = {
    'memory': dict(mem_length=2, mem_delay=2),
    'password': dict(password_length=5),
    'stochastic': dict(p=0.7, horizon=100),
    'bandit': dict(num_actions=10, reward_scale=1, reward_noise=1),
}


class NumpyLegacyRandom:
    """The parts of numpy's legacy ``RandomState`` the ocean envs use."""

    def __init__(self):
        self.mt = MT19937()
        self.mt.init_genrand(0)
        self.has_gauss, self.gauss = False, 0.0

    def seed(self, s):
        s = int(s)
        if not 0 <= s < 2 ** 32:
            raise ValueError('Seed must be between 0 and 2**32 - 1')
        self.mt.init_genrand(s)
        self.has_gauss, self.gauss = False, 0.0

    def randint(self, high):
        """randint(0, high) for one int64 value: masked rejection (legacy buffered_bounded_masked_uint32)."""
        rng = high - 1
        if rng == 0:
            return 0
        mask = rng
        for sh in (1, 2, 4, 8, 16):
            mask |= mask >> sh
        while True:
            v = self.mt.genrand_uint32() & mask
            if v <= rng:
                return v

    def legacy_double(self):
        a = self.mt.genrand_uint32() >> 5
        b = self.mt.genrand_uint32() >> 6
        return (a * 67108864.0 + b) / 9007199254740992.0

    def randn(self):
        if self.has_gauss:
            self.has_gauss = False
            g, self.gauss = self.gauss, 0.0
            return g
        while True:
            x1 = 2.0 * self.legacy_double() - 1.0
            x2 = 2.0 * self.legacy_double() - 1.0
            r2 = x1 * x1 + x2 * x2
            if r2 < 1.0 and r2 != 0.0:
                break
        f = math.sqrt(-2.0 * math.log(r2) / r2)
        self.gauss, self.has_gauss = f * x1, True
        return f * x2


class OceanSerial:
    """``vector.Serial`` over N envs of one ocean kind; recv() returns the buffers like Serial.recv."""

    def __init__(self, kind, num_envs, index_offset=0, **kwargs):
        params = dict(DEFAULTS[kind])
        params.update(kwargs)
        self.kind, self.n, self.index_offset = kind, num_envs, index_offset
        self.rng = NumpyLegacyRandom()                           # the process-global np.random
        n = num_envs
        if kind == 'memory':
            self.L, self.D = int(params['mem_length']), int(params['mem_delay'])
            self.h = 2 * self.L + self.D
            obs_len = 1
        elif kind == 'password':
            self.L = int(params['password_length'])
            obs_len = self.L
        elif kind == 'stochastic':
            self.p, self.horizon = params['p'], 100              # environment.py:67-68 passes horizon=100
            obs_len = 1
        else:
            self.n_act, self.scale, self.noise = params['num_actions'], params['reward_scale'], params['reward_noise']
            obs_len = 1
        self.observations = np.zeros((n, obs_len), dtype=np.float32)
        self.rewards = np.zeros(n, dtype=np.float32)
        self.terminals = np.zeros(n, dtype=bool)
        self.truncations = np.zeros(n, dtype=bool)
        self.masks = np.ones(n, dtype=bool)
        self.agent_ids = np.arange(n)
        self.done = np.ones(n, dtype=bool)
        self.tick = np.zeros(n, dtype=np.int64)
        self.state = [None] * n                                  # per-env solution / count / submission
        self.ep = [None] * n                                     # EpisodeStats.info
        self.infos = []

    # -- Env.reset / Env.step -------------------------------------------------------------------------------------
    def _reset_env(self, i, seed):
        k, rng = self.kind, self.rng
        if k in ('password', 'bandit'):
            seed = 42                                            # hard_fixed_seed
        if seed is not None:
            rng.seed(seed)
        if k == 'memory':                                        # ocean.py:87-97
            sol = np.array([rng.mt.genrand_uint32() & 1 for _ in range(self.h)], dtype=np.float32)
            sol[-(self.L + self.D):] = -1
            self.state[i] = [sol, np.zeros(self.h) - 1]
            self.tick[i] = 1
            self.observations[i, 0] = sol[0]
        elif k == 'password':                                    # ocean.py:251-264
            self.observations[i] = -1
            self.state[i] = np.array([rng.mt.genrand_uint32() & 1 for _ in range(self.L)], dtype=np.float32)
            self.tick[i] = 0
        elif k == 'stochastic':                                  # ocean.py:551-560
            self.tick[i] = 0
            self.state[i] = 0
            self.observations[i] = 0
        else:                                                    # ocean.py:33-44
            self.state[i] = rng.randint(self.n_act)
            self.observations[i] = 1
        self.ep[i] = dict(episode_return=[], episode_length=0)
        self.done[i] = False
        self.rewards[i] = 0
        self.terminals[i] = False
        self.truncations[i] = False
        self.masks[i] = True

    def _step_env(self, i, action):
        k, a, info = self.kind, int(action), {}
        if k == 'memory':                                        # ocean.py:99-123
            sol, sub = self.state[i]
            t = int(self.tick[i])
            ob = reward = 0.0
            if t < self.L:
                ob = sol[t]
                reward = float(a == 0)
            if t >= self.L + self.D:
                s = sol[t - self.L - self.D]
                reward = float(a == s)
                sub[t] = a
            self.tick[i] = t + 1
            terminal = self.tick[i] == self.h
            if terminal:
                info['score'] = np.all(sol[:self.L] == sub[-self.L:])
            self.observations[i, 0] = ob
        elif k == 'password':                                    # ocean.py:266-281
            t = int(self.tick[i])
            self.observations[i, t] = a
            self.tick[i] = t + 1
            reward = 0
            terminal = self.tick[i] == self.L
            if terminal:
                reward = float(np.all(self.observations[i] == self.state[i]))
                info['score'] = reward
        elif k == 'stochastic':                                  # ocean.py:562-582
            self.tick[i] += 1
            self.state[i] += a == 0
            t, c = int(self.tick[i]), int(self.state[i])
            terminal = t == self.horizon
            frac = c / t
            prox = 1 - (self.p - frac) ** 2
            reward = prox if ((a == 0 and frac < self.p) or (a == 1 and frac >= self.p)) else 0
            if terminal:
                info['score'] = prox
            self.observations[i] = 0
        else:                                                    # ocean.py:46-62
            correct = a == self.state[i]
            reward = 1 if correct else 0
            noise = 0
            if self.noise != 0:
                noise = self.rng.randn() * self.scale
            reward = (reward + noise) * self.scale
            terminal = True
            info['score'] = correct
        ep = self.ep[i]                                          # postprocess.py:22-54
        for key, v in info.items():
            ep.setdefault(key, []).append(v)
        ep['episode_return'].append(reward)
        ep['episode_length'] += 1
        self.rewards[i] = reward
        self.terminals[i] = terminal
        self.truncations[i] = False
        self.masks[i] = True
        self.done[i] = terminal
        if terminal:
            return {'episode_return': sum(ep['episode_return']), 'episode_length': ep['episode_length'],
                    'score': float(sum(ep['score']))}
        return {}

    # -- vector.Serial ----------------------------------------------------------------------------------------------
    def async_reset(self, seed=42):
        self.infos = []
        for i in range(self.n):
            self._reset_env(i, seed + self.index_offset + i)

    def send(self, actions):
        actions = np.asarray(actions)
        self.infos = []
        for i in range(self.n):
            if self.done[i]:
                self._reset_env(i, None)
                info = {}
            else:
                info = self._step_env(i, actions[i])
            if info:
                self.infos.append(info)

    def recv(self):
        return (self.observations, self.rewards, self.terminals, self.truncations, self.infos, self.agent_ids,
                self.masks)


class OceanMultiprocessing:
    """``vector.Multiprocessing`` in its synchronous mode (batch_size == num_envs): one Serial per worker, each with
    its own process-global np.random, seeds sliced per worker (vector.py:168-190, 424-428); rows and infos in worker
    order."""

    def __init__(self, kind, num_envs, num_workers, **kwargs):
        assert num_envs % num_workers == 0
        e = num_envs // num_workers
        self.workers = [OceanSerial(kind, e, index_offset=w * e, **kwargs) for w in range(num_workers)]
        self.n, self.e = num_envs, e
        self.agent_ids = np.arange(num_envs)

    def async_reset(self, seed=42):
        for w in self.workers:
            w.async_reset(seed)

    def send(self, actions):
        actions = np.asarray(actions)
        for k, w in enumerate(self.workers):
            w.send(actions[k * self.e:(k + 1) * self.e])

    def recv(self):
        cat = lambda name: np.concatenate([getattr(w, name) for w in self.workers])   # noqa: E731
        infos = [i for w in self.workers for i in w.infos]
        return (cat('observations'), cat('rewards'), cat('terminals'), cat('truncations'), infos, self.agent_ids,
                cat('masks'))
