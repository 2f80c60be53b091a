"""The Atari preprocessing layer of the pixel kinds (oracle/SPEC_PIXEL_PREPROCESSING.md) over the unchanged game oracles:
``OracleVec('pong')`` and ``BreakoutPixelsVec``, one single-env instance per env (``env_index_offset = offset + e``), so each
env stops its frame skip on its own.  Every tick is one send of the plain oracle; this layer restates the no-op draw, the
early stop, the max-pooling (a literal ``np.maximum`` of the last two tick frames), the clip, the soft reset and the
EpisodeStats.  TEST INFRASTRUCTURE (see oracle/__init__.py).  API mirrors vector.Serial: async_reset / send / recv."""
import numpy as np

from .breakout_pixels import BreakoutPixelsVec
from .envs import OracleVec

OBS_SHAPE = (4, 84, 84)
NUM_ACTIONS = {'pong': 6, 'breakout_pixels': 4}
NOOP = 0
M64 = (1 << 64) - 1


def mix32(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return (x ^ (x >> 31)) >> 32


def noop_count(seed_e, k, noop_max):
    """NOOP ticks after real reset number k (from 0) of the env with seed seed_e; 0 when noop_max = 0."""
    if noop_max == 0:
        return 0
    r = mix32((((seed_e ^ 0x6E6F6F705F726E64) * 0x9E3779B97F4A7C15) + k * 0xD1B54A32D192ED03) & M64)
    return 1 + r % noop_max


class _Game:
    """One env of the plain oracle, driven one tick at a time."""

    def __init__(self, kind, env_index, iparam):
        self.kind = kind
        if kind == 'pong':
            self.g = OracleVec('pong', 1, env_index_offset=env_index, iparam=iparam)
        else:
            self.g = BreakoutPixelsVec(1, env_index_offset=env_index, iparam=iparam)
        self.g.collect_infos = False

    def frame(self):
        return self.g.observations[0, 3].copy()

    def lives(self):
        return int(round(float(self.g.state.observations[0, 5]) * 8)) if self.kind == 'breakout_pixels' else 0

    def reset(self, seed=None):
        """async_reset(seed), or (seed None) the plain game's reset row after a game ended."""
        if seed is None:
            self.g.send(np.zeros(1, dtype=np.int64))
        else:
            self.g.async_reset(seed)

    def tick(self, action):
        """-> (reward, game ended)"""
        self.g.send(np.array([action], dtype=np.int64))
        _, r, term = self.g.recv()[:3]
        return float(r[0]), bool(term[0])

    def stats(self):
        s = self.g.state if self.kind == 'breakout_pixels' else self.g
        return float(s.info_return[0]), int(s.info_length[0]), float(s.info_score[0])

    def close(self):
        self.g.close()


class PreprocessedVec:
    def __init__(self, kind, num_envs, env_index_offset=0, iparam=(), frameskip=1, noop_max=0, episodic_life=False,
                 clip_rewards=False):
        self.kind, self.n = kind, num_envs
        self.offset = env_index_offset
        self.frameskip, self.noop_max = frameskip, noop_max
        self.episodic_life, self.clip_rewards = bool(episodic_life), bool(clip_rewards)
        self.envs = [_Game(kind, env_index_offset + e, iparam) for e in range(num_envs)]
        self.observations = np.zeros((num_envs, *OBS_SHAPE), dtype=np.uint8)
        self.rewards = np.zeros(num_envs, dtype=np.float32)
        self.terminals = np.zeros(num_envs, dtype=bool)
        self.truncations = np.zeros(num_envs, dtype=bool)
        self.masks = np.ones(num_envs, dtype=bool)
        self.ended = np.zeros(num_envs, dtype=bool)      # the row ended a game
        self.soft = np.zeros(num_envs, dtype=bool)       # a soft reset is pending
        self.resets = np.zeros(num_envs, dtype=np.int64)  # real resets since async_reset (the no-op draw key)
        self.noops = []                                   # (env, no-op ticks) of every real reset, for the tests
        self.agent_ids = np.arange(num_envs)
        self.infos = []
        self.collect_infos = True
        self.seed = 0

    def _real_reset(self, e, seed=None):
        g = self.envs[e]
        g.reset(seed)
        n = noop_count((self.seed + self.offset + e) & M64, int(self.resets[e]), self.noop_max)
        for _ in range(n):
            _, end = g.tick(NOOP)
            assert not end, 'no-op ticks never end a game'
        self.noops.append((e, n))
        self.resets[e] += 1
        self.observations[e] = g.frame()[None]

    def _skip(self, e, action):
        """Up to frameskip ticks of `action`, stopping where the game ends -> (reward sum, game ended, max frame)."""
        g = self.envs[e]
        frames, total, end = [], 0.0, False
        for _ in range(self.frameskip):
            r, end = g.tick(action)
            total += r
            frames.append(g.frame())
            if end:
                break
        frame = frames[-1] if len(frames) == 1 else np.maximum(frames[-2], frames[-1])
        return total, end, frame

    def async_reset(self, seed=42):
        self.seed = seed % (1 << 64)
        self.resets[:] = 0
        self.soft[:] = False
        for e in range(self.n):
            self._real_reset(e, self.seed)
        self.rewards[:] = 0
        self.terminals[:] = False
        self.ended[:] = False
        self.infos = []

    def send(self, actions):
        actions = np.asarray(actions, dtype=np.int64)
        infos = []
        for e in range(self.n):
            g = self.envs[e]
            if self.terminals[e] and not self.soft[e]:
                self._real_reset(e)
                self.rewards[e], self.terminals[e], self.ended[e] = 0, False, False
                continue
            if self.terminals[e]:        # soft reset: one no-op step, all 4 slots; terminal only if the game ended
                self.soft[e] = False
                _, end, frame = self._skip(e, NOOP)
                self.observations[e] = frame[None]
                self.rewards[e], self.terminals[e], self.ended[e] = 0, end, end
            else:
                lives0 = g.lives()
                total, end, frame = self._skip(e, int(actions[e]))
                lost = self.episodic_life and 0 < g.lives() < lives0
                self.observations[e, :3] = self.observations[e, 1:].copy()
                self.observations[e, 3] = frame
                self.rewards[e] = np.sign(total) if self.clip_rewards else total
                self.terminals[e], self.ended[e] = end or lost, end
                self.soft[e] = lost and not end
            if self.ended[e]:
                ret, length, score = g.stats()
                infos.append({'episode_return': ret, 'episode_length': length, 'score': score})
        self.infos = infos if self.collect_infos else []

    def recv(self):
        return (self.observations, self.rewards, self.terminals, self.truncations, self.infos, self.agent_ids,
                self.masks)

    def close(self):
        for g in self.envs:
            g.close()
        self.envs = []
