"""Host-side structured-observation layout vs the reference's own known-answer vectors
(reference tests/test_pytorch.py:14-134, copied here as expected VALUES -- they are test data, not code) and vs
numpy's aligned-struct rules (pufferlib/emulation.py:68-80)."""
import numpy as np
import pytest
import torch

from pufferlib_b200 import emulation, spaces
from pufferlib_b200.namespace import namespace

CASES = [
    (np.dtype((np.uint8, (4,)), align=True), np.dtype([('x', np.uint8, (4,))], align=True),
     {'x': (torch.uint8, (4,), 0, 4)}),
    (np.dtype((np.uint8, (4, 5)), align=True), np.dtype([('x', np.uint8, (4, 5))], align=True),
     {'x': (torch.uint8, (4, 5), 0, 20)}),
    (np.dtype((np.uint8, (4,)), align=True), np.dtype([('x', np.uint32, (1,))], align=True),
     {'x': (torch.uint32, (1,), 0, 4)}),
    (np.dtype((np.uint8, (12,)), align=True), np.dtype([('foo', np.int32, (1,)), ('bar', np.int32, (2,))], align=True),
     {'foo': (torch.int32, (1,), 0, 4), 'bar': (torch.int32, (2,), 4, 8)}),
    (np.dtype((np.uint8, (16,)), align=True),
     np.dtype([('foo', np.int32, (1,)), ('bar', [('a', np.int32, (2,)), ('b', np.int32, (1,))])], align=True),
     {'foo': (torch.int32, (1,), 0, 4), 'bar': {'a': (torch.int32, (2,), 4, 8), 'b': (torch.int32, (1,), 12, 4)}}),
    (np.dtype((np.float32, (4,)), align=True),
     np.dtype([('foo', np.float32, (1,)), ('bar', [('a', np.float32, (2,)), ('b', np.float32, (1,))])], align=True),
     {'foo': (torch.float32, (1,), 0, 1), 'bar': {'a': (torch.float32, (2,), 1, 2), 'b': (torch.float32, (1,), 3, 1)}}),
    (np.dtype((np.int32, (4,)), align=True),
     np.dtype([('foo', np.int32, (1,)),
               ('bar', [('a', [('y', np.int32, (1,)), ('z', np.int32, (1,))]), ('b', np.int32, (1,))])], align=True),
     {'foo': (torch.int32, (1,), 0, 1),
      'bar': {'a': {'y': (torch.int32, (1,), 1, 1), 'z': (torch.int32, (1,), 2, 1)}, 'b': (torch.int32, (1,), 3, 1)}}),
    # alignment padding: uint8(7,7)@8 ends at 57, int32(2,3) starts at 60, record = 84 bytes
    (np.dtype((np.uint8, (84,)), align=True),
     np.dtype([('xx', np.float32, (1, 2)), ('yy', [('aa', np.uint8, (7, 7)), ('bb', np.int32, (2, 3))])], align=True),
     {'xx': (torch.float32, (1, 2), 0, 8),
      'yy': {'aa': (torch.uint8, (7, 7), 8, 49), 'bb': (torch.int32, (2, 3), 60, 24)}}),
]


@pytest.mark.parametrize('observation_dtype,emulated_dtype,expected', CASES)
def test_nativize_dtype_known_answers(observation_dtype, emulated_dtype, expected):
    got = emulation.nativize_dtype(namespace(observation_dtype=observation_dtype,
                                             emulated_observation_dtype=emulated_dtype))
    assert got == expected


def nested_space():
    return spaces.Dict({'x': spaces.Box(-1.0, 1.0, (1, 2), np.float32),
                        'y': spaces.Dict({'a': spaces.Box(0, 255, (7, 7), np.uint8),
                                          'b': spaces.Box(-1024, 1024, (2, 3), np.int32)})})


def test_dtype_from_space_and_flat_space():
    sp = nested_space()
    dt = emulation.dtype_from_space(sp)
    assert dt.itemsize == 84 and dt.isalignedstruct
    assert dt.fields['y'][0].fields['b'][1] == 52 and dt.fields['y'][1] == 8        # bb at 8+52 = 60
    flat, struct = emulation.emulate_observation_space(sp)
    assert flat.shape == (84,) and flat.dtype == np.uint8 and struct == dt
    same = spaces.Dict({'xx': spaces.Box(-1, 1, (1, 2), np.float32), 'yy': spaces.Box(-1, 1, (4, 5), np.float32)})
    flat2, _ = emulation.emulate_observation_space(same)
    assert flat2.shape == (22,) and flat2.dtype == np.float32                       # common leaf dtype is kept
    box = spaces.Box(0, 1, (3,), np.float32)
    assert emulation.emulate_observation_space(box)[0] is box
    tup = spaces.Tuple([spaces.Discrete(3), spaces.Box(0, 1, (2,), np.float32)])
    assert emulation.dtype_from_space(tup).names == ('f0', 'f1')
    leaves = emulation.leaf_layout(dt)
    assert [(p, o, n) for p, _, _, o, n in leaves] == [(('x',), 0, 8), (('y', 'a'), 8, 49), (('y', 'b'), 60, 24)]


def test_nativize_tensor_roundtrip_cpu():
    """emulate (numpy structured assignment) -> nativize_tensor views, like test_pytorch.py:137-211."""
    sp = nested_space()
    dt = emulation.dtype_from_space(sp)
    flat_space, _ = emulation.emulate_observation_space(sp)
    native = emulation.nativize_dtype(namespace(observation_dtype=np.dtype(np.uint8), emulated_observation_dtype=dt))
    rng = np.random.default_rng(0)
    n = 5
    rec = np.zeros(n, dtype=dt)
    rec['x'] = rng.standard_normal((n, 1, 2)).astype(np.float32)
    rec['y']['a'] = rng.integers(0, 256, (n, 7, 7), dtype=np.uint8)
    rec['y']['b'] = rng.integers(-1024, 1024, (n, 2, 3), dtype=np.int32)
    obs = torch.from_numpy(rec.view(np.uint8).reshape(n, -1))
    views = emulation.nativize_tensor(obs, native)
    assert np.array_equal(views['x'].numpy(), rec['x'])
    assert np.array_equal(views['y']['a'].numpy(), rec['y']['a'])
    assert np.array_equal(views['y']['b'].numpy(), rec['y']['b'])
