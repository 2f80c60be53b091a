"""ctypes front-end of ``oracle/csrc/pong_versus.c``: a Serial-like vectoriser over two-player pong from pixels
(oracle/SPEC_PONG_VERSUS.md), two agent rows per env, driven the way ``vector.Serial`` drives a PettingZoo env.
TEST INFRASTRUCTURE (see oracle/__init__.py).  API mirrors vector.Serial: async_reset / send / recv.

Infos: for every env whose game ended on this send, in env order, the env's per-agent info dict (MultiagentEpisodeStats
passes it through unchanged, reference postprocess.py:147-179): {1: {'score': s, 'episode_length': L},
2: {'score': -s, 'episode_length': L}} with s = agent 1's (the right paddle's) points minus agent 2's and L the game's
ticks."""
import ctypes as C

import numpy as np

from . import build as _build

NUM_ACTIONS = 6
AGENTS = 2


def _lib():
    lib = _build.load()
    if not getattr(lib, '_pv_typed', False):
        lib.oracle_pv_create.restype = C.c_void_p
        lib.oracle_pv_create.argtypes = [C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int]
        lib.oracle_pv_destroy.argtypes = [C.c_void_p]
        lib.oracle_pv_reset.argtypes = [C.c_void_p, C.c_uint64] + [C.c_void_p] * 3
        lib.oracle_pv_step.argtypes = [C.c_void_p] + [C.c_void_p] * 6
        lib._pv_typed = True
    return lib


class PongVersusVec:
    def __init__(self, num_envs, framestack=4, env_index_offset=0, max_score=0, max_ticks=0):
        self.lib = _lib()
        self.n, self.S = num_envs, framestack
        self.h = C.c_void_p(self.lib.oracle_pv_create(num_envs, env_index_offset, framestack, max_score, max_ticks))
        assert self.h
        rows = AGENTS * num_envs
        self.observations = np.zeros((rows, framestack, 84, 84), dtype=np.uint8)
        self.rewards = np.zeros(rows, dtype=np.float32)
        self.terminals = np.zeros(rows, dtype=bool)
        self.truncations = np.zeros(rows, dtype=bool)
        self.masks = np.ones(rows, dtype=bool)
        self.info_score = np.zeros(num_envs, dtype=np.int32)
        self.info_length = np.zeros(num_envs, dtype=np.int32)
        self.agent_ids = np.arange(rows)
        self.infos = []

    def _p(self, a):
        return a.ctypes.data_as(C.c_void_p)

    def async_reset(self, seed=42):
        self.lib.oracle_pv_reset(self.h, C.c_uint64(seed % (1 << 64)), self._p(self.observations),
                                 self._p(self.rewards), self._p(self.terminals))
        self.infos = []

    def send(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.int64)
        assert a.shape == (AGENTS * self.n,)
        self.lib.oracle_pv_step(self.h, self._p(a), self._p(self.observations), self._p(self.rewards),
                                self._p(self.terminals), self._p(self.info_score), self._p(self.info_length))
        ended = self.terminals.reshape(-1, AGENTS).all(axis=1)
        self.infos = [{1: {'score': int(self.info_score[e]), 'episode_length': int(self.info_length[e])},
                       2: {'score': -int(self.info_score[e]), 'episode_length': int(self.info_length[e])}}
                      for e in np.nonzero(ended)[0]]

    def recv(self):
        return (self.observations, self.rewards, self.terminals, self.truncations, self.infos, self.agent_ids,
                self.masks)

    def close(self):
        if self.h:
            self.lib.oracle_pv_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
