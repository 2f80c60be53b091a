"""``vector.Serial`` over N ``Squared`` envs, restated as one array program.  TEST INFRASTRUCTURE.

Follows (all under reference pufferlib/):
  environments/ocean/ocean.py:424        MOVES table
  environments/ocean/ocean.py:444-446    _all_possible_targets (x-major perimeter order)
  environments/ocean/ocean.py:448-463    Squared.reset  (grid=0, agent -1 at centre, one target +1)
  environments/ocean/ocean.py:465-513    Squared.step   (reward before target removal / teleport)
  environments/ocean/environment.py:28-31  make_squared defaults distance_to_target=3, num_targets=1
  postprocess.py:8-54                    EpisodeStats (episode_return = python-float sum, episode_length, score)
  emulation.py:169-194, 196-228          GymnasiumPufferEnv reset/step -> buf rows (r=0,d=F,t=F,mask=T on reset)
  vector.py:112-162, 639-641             Serial.async_reset / send / recv, make_seeds = seed + i

RNG: one process-global MT19937 (oracle/mt19937.py).  ``async_reset(seed)`` re-seeds it per env with
``seed + i`` and takes one ``randbelow(8 d)``; every later auto-reset (``env.reset()`` with seed None,
vector.py:147-149) draws the next ``randbelow`` from the stream left by the LAST seeded env, in env order.
Only ``num_targets == 1`` is restated (the reference default; ``random.sample(pop, 1)`` == one randbelow).
"""
import numpy as np

from .mt19937 import MT19937

MOVES = [(0, -1), (0, 1), (-1, 0), (1, 0), (1, -1), (-1, -1), (1, 1), (-1, 1)]


def possible_targets(grid_size):
    g = grid_size
    return [(x, y) for x in range(g) for y in range(g) if x == 0 or y == 0 or x == g - 1 or y == g - 1]


def reward_table(distance_to_target):
    """fp32(1 - k/d) for k = 0..2d: python-double arithmetic then the fp32 store of emulation.py:221."""
    d = distance_to_target
    return np.array([1 - k / d for k in range(2 * d + 1)], dtype=np.float64).astype(np.float32)


class SquaredSerial:
    def __init__(self, num_envs, distance_to_target=3, num_targets=1, index_offset=0):
        assert num_targets == 1, 'oracle restates the num_targets=1 path only'
        self.index_offset = index_offset      # global index of env 0 (a Multiprocessing worker's slice of the seeds)
        self.n = num_envs
        self.d = distance_to_target
        self.g = 2 * distance_to_target + 1
        self.max_ticks = num_targets * distance_to_target
        self.targets_all = possible_targets(self.g)
        self.rng = MT19937(0)  # EpisodeStats.__init__ resets unseeded (postprocess.py:15); reseeded below
        n, g = self.n, self.g
        self.observations = np.zeros((n, g, g), dtype=np.float32)
        self.rewards = np.zeros(n, dtype=np.float32)
        self.terminals = np.zeros(n, dtype=bool)
        self.truncations = np.zeros(n, dtype=bool)
        self.masks = np.ones(n, dtype=bool)
        self.agent_ids = np.arange(n)
        self.pos = np.zeros((n, 2), dtype=np.int64)
        self.tick = np.zeros(n, dtype=np.int64)
        self.target = np.zeros((n, 2), dtype=np.int64)
        self.hit = np.zeros(n, dtype=bool)
        self.done = np.ones(n, dtype=bool)
        self.ep_rewards = [[] for _ in range(n)]
        self.infos = []

    def _reset_env(self, i, seed):
        if seed is not None:
            self.rng.seed(seed)                                   # ocean.py:449-451
        d = self.d
        self.observations[i] = 0
        self.observations[i, d, d] = -1
        self.pos[i] = (d, d)
        self.tick[i] = 0
        j = self.rng.randbelow(len(self.targets_all))             # random.sample(pop, 1)  ocean.py:459
        self.target[i] = self.targets_all[j]
        self.observations[i, self.target[i, 0], self.target[i, 1]] = 1
        self.hit[i] = False
        self.done[i] = False
        self.ep_rewards[i] = []
        self.rewards[i] = 0                                       # emulation.py:187-192
        self.terminals[i] = False
        self.truncations[i] = False
        self.masks[i] = True

    def async_reset(self, seed=42):
        self.infos = []
        for i in range(self.n):
            self._reset_env(i, seed + self.index_offset + i)      # vector.py:639-641 (424-428: a worker gets its slice)

    def _step_env(self, i, action):
        d = self.d
        x, y = int(self.pos[i, 0]), int(self.pos[i, 1])         # python ints: reward is a python float
        self.observations[i, x, y] = 0
        dx, dy = MOVES[int(action)]
        x += dx
        y += dy
        tx, ty = int(self.target[i, 0]), int(self.target[i, 1])
        min_dist = max(abs(x - tx), abs(y - ty))                  # single target; removed only on the done step
        reward = 1 - min_dist / d                                 # python double
        if (x, y) == (tx, ty):
            self.hit[i] = True
        if max(abs(x - d), abs(y - d)) >= d:
            self.pos[i] = (d, d)
        else:
            self.pos[i] = (x, y)
        self.observations[i, self.pos[i, 0], self.pos[i, 1]] = -1
        self.tick[i] += 1
        done = bool(self.tick[i] >= self.max_ticks)
        self.ep_rewards[i].append(reward)
        self.rewards[i] = reward
        self.terminals[i] = done
        self.truncations[i] = False
        self.masks[i] = True
        self.done[i] = done
        if done:
            return {'episode_return': sum(self.ep_rewards[i]),    # builtin sum of python floats (compensated in CPython>=3.12), postprocess.py:38-40
                    'episode_length': len(self.ep_rewards[i]),
                    'score': 1.0 if self.hit[i] else 0.0}          # (num_targets - len(targets)) / num_targets
        return {}

    def send(self, actions):
        actions = np.asarray(actions)
        self.infos = []
        for i in range(self.n):
            if self.done[i]:
                self._reset_env(i, None)                          # vector.py:147-149 (action ignored)
                info = {}
            else:
                info = self._step_env(i, actions[i])
            if info:
                self.infos.append(info)

    def recv(self):
        return (self.observations, self.rewards, self.terminals, self.truncations,
                self.infos, self.agent_ids, self.masks)


class SquaredMultiprocessing:
    """``vector.Multiprocessing`` (synchronous mode, batch_size == num_envs) over ``Squared``: every worker process is a
    ``Serial`` over its own envs with its OWN process-global MT19937 (vector.py:168-190, seeds sliced per worker at
    :424-428), so auto-resets draw from the stream left by the worker's last seeded env, in env order inside the worker.
    recv() returns the workers' rows in worker order (vector.py:360-369); infos likewise (:397-401)."""

    def __init__(self, num_envs, num_workers, distance_to_target=3):
        assert num_envs % num_workers == 0
        e = num_envs // num_workers
        self.workers = [SquaredSerial(e, distance_to_target, index_offset=w * e) for w in range(num_workers)]
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
