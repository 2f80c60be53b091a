"""breakout_pixels without a device: the oracle's C renderer (oracle/csrc/breakout_pixels.c, behind
oracle/breakout_pixels.py) against an independent numpy restatement of oracle/SPEC_BREAKOUT_PIXELS.md applied to the
`breakout` oracle's rows of the same game, and how the creator resolves."""
import numpy as np
import pytest

from oracle.breakout_pixels import BreakoutPixelsVec
from oracle.envs import OracleVec
from pufferlib_b200.environments import ocean, resolve, resolve_config
from pufferlib_b200.exceptions import APIUsageError

# field rectangle of every frame row / column: [LO, HI)
Y_LO, Y_HI = (200 * np.arange(84)) // 84, (200 * np.arange(1, 85)) // 84
X_LO, X_HI = (160 * np.arange(84)) // 84, (160 * np.arange(1, 85)) // 84
GRAY = np.array([176, 160, 144, 128, 112, 96], dtype=np.uint8)


def field_from_state_row(o):
    """The 200 x 160 field of one `breakout` observation row (px, bx, by and the brick bitmap are exact in it)."""
    px, bx, by = (int(round(float(v) * 256)) for v in o[:3])
    f = np.zeros((200, 160), dtype=np.uint8)
    alive = o[8:128].reshape(6, 20) > 0
    for row in range(6):
        for col in range(20):
            if alive[row, col]:
                f[30 + 6 * row:36 + 6 * row, 8 * col:8 * col + 8] = GRAY[row]
    f[190:192, px:px + 24] = 192
    f[by:by + 2, bx:bx + 2] = 255
    return f


def frame_from_field(f):
    """Frame pixel (r, c) = max of the field over its rectangle: np.maximum.reduceat over the row then column bounds."""
    rows = np.maximum.reduceat(f, Y_LO, axis=0)
    return np.maximum.reduceat(rows, X_LO, axis=1)


def test_rectangles_tile_the_field():
    assert Y_LO[0] == 0 and Y_HI[-1] == 200 and np.array_equal(Y_LO[1:], Y_HI[:-1])
    assert X_LO[0] == 0 and X_HI[-1] == 160 and np.array_equal(X_LO[1:], X_HI[:-1])
    assert set(Y_HI - Y_LO) == {2, 3} and set(X_HI - X_LO) == {1, 2}


def run_pair(n, h, seed, max_ticks=None, offset=0):
    """Drive the oracle's breakout and breakout_pixels with one seed and action tape; every pixel row must equal the
    numpy frame stack built from the breakout rows, and rewards / terminals / infos must be the same."""
    ip = [max_ticks] if max_ticks else []
    state = OracleVec('breakout', n, env_index_offset=offset, iparam=ip)
    pix = BreakoutPixelsVec(n, env_index_offset=offset, iparam=ip)
    # FIRE-heavy tape so balls launch early and bricks fall; LEFT / RIGHT so lives are lost
    tape = np.random.default_rng(seed).choice(4, size=(h, n), p=[0.2, 0.3, 0.25, 0.25]).astype(np.int64)
    state.async_reset(seed)
    pix.async_reset(seed)
    stack = np.zeros((n, 4, 84, 84), dtype=np.uint8)
    done = np.ones(n, dtype=bool)
    counts = dict(resets=0, life_losses=0, bricks=0, terminals=0)
    lives_prev = np.zeros(n)
    for t in range(h + 1):
        so, sr, st, _, sinf, _, _ = state.recv()
        po, pr, pt, _, pinf, _, _ = pix.recv()
        for i in range(n):
            frame = frame_from_field(field_from_state_row(so[i]))
            if done[i]:
                stack[i] = frame
                counts['resets'] += 1
            else:
                stack[i, :3] = stack[i, 1:]
                stack[i, 3] = frame
                counts['life_losses'] += int(so[i][5] * 8 < lives_prev[i])
            lives_prev[i] = so[i][5] * 8
        assert np.array_equal(po, stack), f'step {t}: frames differ in envs {np.nonzero((po != stack).any((1, 2, 3)))[0]}'
        assert np.array_equal(pr.view(np.uint32), sr.view(np.uint32)) and np.array_equal(pt, st), t
        assert pinf == sinf, t
        # every object is visible in every frame: the ball (255) and the paddle (192)
        assert (po[:, 3] == 255).any((1, 2)).all() and (po[:, 3] == 192).any((1, 2)).all(), t
        counts['bricks'] += int((sr > 0).sum())
        counts['terminals'] += int(st.sum())
        done = st.copy()
        if t < h:
            state.send(tape[t])
            pix.send(tape[t])
    state.close()
    pix.close()
    return counts


@pytest.mark.parametrize('n,h,seed,max_ticks,offset', [(7, 600, 1, 250, 0), (5, 700, 2, None, 3)])
def test_oracle_pixels_equal_numpy_render_of_breakout(n, h, seed, max_ticks, offset):
    """Long enough for bricks to fall and lives to be lost (with max_ticks, episodes also end and reset)."""
    c = run_pair(n, h, seed, max_ticks, offset)
    assert c['life_losses'] > 0 and c['bricks'] > 0, c
    if max_ticks:
        assert c['terminals'] > 0 and c['resets'] > n, c


def test_oracle_pixels_short_episodes():
    """Many reset rows: 33 envs, 40-tick episodes, a nonzero env_index_offset."""
    c = run_pair(33, 160, 3, 40, 1000)
    assert c['terminals'] >= 3 * 33 and c['resets'] >= 4 * 33, c


def test_creator_resolution():
    c = ocean.env_creator('breakout_pixels')
    assert c.__name__ == 'make_breakout_pixels' and c is ocean.make_breakout_pixels
    assert resolve_config(c, [], {}) == ('breakout_pixels', [0] * 8, [])
    assert resolve(c, [], {'max_ticks': 500}) == ('breakout_pixels', [500] + [0] * 7)
    assert resolve(c, [], {'max_ticks': 65535})[1][0] == 65535

    def make_breakout_pixels(max_ticks=4096):      # recognised by name, like the other kinds
        pass
    assert resolve(make_breakout_pixels, [], {'max_ticks': 7})[0] == 'breakout_pixels'
    with pytest.raises(APIUsageError):
        c()                                           # device-native: no CPU instance


@pytest.mark.parametrize('kwargs', [{'max_ticks': 0}, {'max_ticks': -5}, {'max_ticks': 65536}, {'max_ticks': 2.5},
                                    {'max_ticks': '100'}, {'max_score': 3}, {'max_ticks': 10, 'frameskip': 4}])
def test_bad_kwargs_refused(kwargs):
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator('breakout_pixels'), [], kwargs)


def test_positional_args_refused():
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator('breakout_pixels'), [100], {})
