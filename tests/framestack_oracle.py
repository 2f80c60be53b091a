"""The pixel kinds with an S-frame observation (the `framestack` keyword, S = 1 or 4): each env's game is one single-env
instance of the unchanged game oracles (oracle/pixel_preprocessing.py's `_Game` over `OracleVec('pong')` and
`BreakoutPixelsVec`), driven one tick at a time under the Atari preprocessing rules of
oracle/SPEC_PIXEL_PREPROCESSING.md, and this class keeps the S frames the way gymnasium's FrameStack does: every slot
filled with the first frame on a reset, the oldest frame dropped and the new one appended on a step.  A soft reset
(episodic_life) is a reset row: its frame fills every slot.  With S = 4 and the default options this is the plain
oracle; the tests check that, and that S = 1 is the newest slot of S = 4.
TEST INFRASTRUCTURE.  API mirrors vector.Serial: async_reset / send / recv."""
import numpy as np

from oracle.pixel_preprocessing import M64, NOOP, _Game, noop_count


class FrameStackVec:
    def __init__(self, kind, num_envs, framestack=4, env_index_offset=0, iparam=(), frameskip=1, noop_max=0,
                 episodic_life=False, clip_rewards=False):
        assert framestack in (1, 4)
        self.kind, self.n, self.S = kind, num_envs, framestack
        self.offset = env_index_offset
        self.frameskip, self.noop_max = frameskip, noop_max
        self.episodic_life, self.clip_rewards = bool(episodic_life), bool(clip_rewards)
        self.envs = [_Game(kind, env_index_offset + e, iparam) for e in range(num_envs)]
        self.observations = np.zeros((num_envs, framestack, 84, 84), dtype=np.uint8)
        self.rewards = np.zeros(num_envs, dtype=np.float32)
        self.terminals = np.zeros(num_envs, dtype=bool)
        self.truncations = np.zeros(num_envs, dtype=bool)
        self.masks = np.ones(num_envs, dtype=bool)
        self.ended = np.zeros(num_envs, dtype=bool)
        self.soft = np.zeros(num_envs, dtype=bool)
        self.resets = np.zeros(num_envs, dtype=np.int64)
        self.agent_ids = np.arange(num_envs)
        self.infos = []
        self.collect_infos = True
        self.seed = 0

    # ---- the frame stack: FrameStack's reset and step
    def _fill(self, e, frame):
        for k in range(self.S):
            self.observations[e, k] = frame

    def _push(self, e, frame):
        for k in range(self.S - 1):
            self.observations[e, k] = self.observations[e, k + 1]
        self.observations[e, self.S - 1] = frame

    # ---- the game under the preprocessing rules
    def _real_reset(self, e, seed=None):
        g = self.envs[e]
        g.reset(seed)
        for _ in range(noop_count((self.seed + self.offset + e) & M64, int(self.resets[e]), self.noop_max)):
            _, end = g.tick(NOOP)
            assert not end
        self.resets[e] += 1
        self._fill(e, g.frame())

    def _skip(self, e, action):
        g = self.envs[e]
        frames, total, end = [], 0.0, False
        for _ in range(self.frameskip):
            r, end = g.tick(action)
            total += r
            frames.append(g.frame())
            if end:
                break
        return total, end, frames[-1] if len(frames) == 1 else np.maximum(frames[-2], frames[-1])

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
            if self.terminals[e]:
                self.soft[e] = False
                _, end, frame = self._skip(e, NOOP)
                self._fill(e, frame)
                self.rewards[e], self.terminals[e], self.ended[e] = 0, end, end
            else:
                lives0 = g.lives()
                total, end, frame = self._skip(e, int(actions[e]))
                lost = self.episodic_life and 0 < g.lives() < lives0
                self._push(e, frame)
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
