"""The breakout_pixels oracle (oracle/SPEC_BREAKOUT_PIXELS.md): the breakout oracle of ``oracle/envs.py`` steps the game,
``oracle/csrc/breakout_pixels.c`` draws each frame from its observation row, and this class keeps the frame stacks.
TEST INFRASTRUCTURE (see oracle/__init__.py).  API mirrors vector.Serial and OracleVec: async_reset / send / recv."""
import ctypes as C

import numpy as np

from . import build as _build
from .envs import OracleVec

OBS_SHAPE = (4, 84, 84)
NUM_ACTIONS = 4


def _lib():
    lib = _build.load()
    if not getattr(lib, '_pixels_typed', False):
        lib.oracle_breakout_pixels_render.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        lib._pixels_typed = True
    return lib


def render(state_rows):
    """[n, 128] float32 breakout observation rows -> [n, 84, 84] uint8 frames."""
    rows = np.ascontiguousarray(state_rows, dtype=np.float32)
    frames = np.zeros((len(rows), 84, 84), dtype=np.uint8)
    _lib().oracle_breakout_pixels_render(rows.ctypes.data_as(C.c_void_p), len(rows), frames.ctypes.data_as(C.c_void_p))
    return frames


class BreakoutPixelsVec:
    def __init__(self, num_envs, env_index_offset=0, iparam=(), threads=None):
        self.state = OracleVec('breakout', num_envs, env_index_offset=env_index_offset, iparam=iparam, threads=threads)
        self.n = num_envs
        self.observations = np.zeros((num_envs, *OBS_SHAPE), dtype=np.uint8)

    @property
    def collect_infos(self):
        return self.state.collect_infos

    @collect_infos.setter
    def collect_infos(self, v):
        self.state.collect_infos = v

    def async_reset(self, seed=42):
        self.state.async_reset(seed)
        self.observations[:] = render(self.state.observations)[:, None]

    def send(self, actions):
        reset = self.state.terminals.copy()        # envs whose previous row was terminal are reset by this send
        self.state.send(actions)
        frames = render(self.state.observations)
        self.observations[:, :3] = self.observations[:, 1:]
        self.observations[:, 3] = frames
        self.observations[reset] = frames[reset][:, None]

    def recv(self):
        o, r, term, trunc, infos, ids, masks = self.state.recv()
        return self.observations, r, term, trunc, infos, ids, masks

    def close(self):
        self.state.close()
