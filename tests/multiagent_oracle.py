"""``vector.Serial`` / ``vector.Multiprocessing`` over the reference's ocean Multiagent env, restated over numpy arrays.
TEST INFRASTRUCTURE (the device kind is checked against it at scale; it is checked against the reference's own
trajectories, tests/golden/multiagent_*.npz).

Follows (all under reference pufferlib/):
  environments/ocean/ocean.py:149-208    Multiagent   (obs {1: [0], 2: [1]}; reward[1] = action[1] == 0,
                                                       reward[2] = action[2] == 1; both agents terminal every step)
  environments/ocean/environment.py:69-72  make_multiagent(): MultiagentEpisodeStats + PettingZooPufferEnv, no args
  postprocess.py:147-179                 MultiagentEpisodeStats (returns the env's infos unchanged)
  emulation.py:236-420                   PettingZooPufferEnv: agent rows in possible_agents order; reset rows r=0,
                                         term=False, trunc=False, mask=True; done = all agents terminal
  vector.py:97-110, 137-156              Serial: agent a of env e at row e*A + a; `if env.done: reset() else: step()`
"""
import numpy as np

AGENTS = (1, 2)


class MultiagentSerial:
    """``vector.Serial`` over N Multiagent envs (2N agent rows); recv() returns the buffers like Serial.recv."""

    def __init__(self, num_envs):
        self.n, a = num_envs, len(AGENTS)
        rows = num_envs * a
        self.observations = np.zeros((rows, 1), dtype=np.float32)
        self.rewards = np.zeros(rows, dtype=np.float32)
        self.terminals = np.zeros(rows, dtype=bool)
        self.truncations = np.zeros(rows, dtype=bool)
        self.masks = np.ones(rows, dtype=bool)
        self.agent_ids = np.arange(rows)
        self.done = np.ones(num_envs, dtype=bool)       # PettingZooPufferEnv.all_done starts True
        self.infos = []

    def _reset_env(self, e):                            # emulation.py:319-347, ocean.py:181-184
        lo = 2 * e
        self.observations[lo:lo + 2, 0] = (0, 1)
        self.rewards[lo:lo + 2] = 0
        self.terminals[lo:lo + 2] = False
        self.truncations[lo:lo + 2] = False
        self.masks[lo:lo + 2] = True
        self.done[e] = False

    def _step_env(self, e, actions):                    # ocean.py:186-208, emulation.py:349-417
        lo = 2 * e
        a1, a2 = int(actions[0]), int(actions[1])
        assert a1 in (0, 1) and a2 in (0, 1)
        reward = {1: 1 if a1 == 0 else 0, 2: 1 if a2 == 1 else 0}
        self.observations[lo:lo + 2, 0] = (0, 1)
        self.rewards[lo:lo + 2] = (reward[1], reward[2])
        self.terminals[lo:lo + 2] = True
        self.truncations[lo:lo + 2] = False
        self.masks[lo:lo + 2] = True
        self.done[e] = True                             # all(dones.values())
        return {1: {'score': reward[1]}, 2: {'score': reward[2]}}

    def async_reset(self, seed=42):                     # Multiagent.reset ignores the seed
        self.infos = []
        for e in range(self.n):
            self._reset_env(e)

    def send(self, actions):
        actions = np.asarray(actions)
        self.infos = []
        for e in range(self.n):
            if self.done[e]:
                self._reset_env(e)                      # reset infos are {}: Serial drops them
            else:
                self.infos.append(self._step_env(e, actions[2 * e:2 * e + 2]))

    def recv(self):
        return (self.observations, self.rewards, self.terminals, self.truncations, self.infos, self.agent_ids,
                self.masks)


class MultiagentMultiprocessing:
    """``vector.Multiprocessing`` in its synchronous mode (batch_size == num_envs): one Serial per worker; rows and infos
    in worker order."""

    def __init__(self, num_envs, num_workers):
        assert num_envs % num_workers == 0
        e = num_envs // num_workers
        self.workers = [MultiagentSerial(e) for _ in range(num_workers)]
        self.rows_per_worker = 2 * e
        self.agent_ids = np.arange(2 * num_envs)

    def async_reset(self, seed=42):
        for w in self.workers:
            w.async_reset(seed)

    def send(self, actions):
        actions = np.asarray(actions)
        k = self.rows_per_worker
        for i, w in enumerate(self.workers):
            w.send(actions[i * k:(i + 1) * k])

    def recv(self):
        cat = lambda name: np.concatenate([getattr(w, name) for w in self.workers])   # noqa: E731
        infos = [i for w in self.workers for i in w.infos]
        return (cat('observations'), cat('rewards'), cat('terminals'), cat('truncations'), infos, self.agent_ids,
                cat('masks'))


def info_rows(t, infos):
    """(recv index, dict index, agent, score) rows of the goldens' info format."""
    return [(t, k, agent, i[agent]['score']) for k, i in enumerate(infos) for agent in sorted(i)]
