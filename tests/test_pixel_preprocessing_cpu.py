"""The Atari preprocessing layer's oracle (oracle/pixel_preprocessing.py, oracle/SPEC_PIXEL_PREPROCESSING.md) against the
plain game oracles it wraps, and the keyword parsing of the pixel kinds: no GPU."""
import numpy as np
import pytest

from oracle.breakout_pixels import BreakoutPixelsVec
from oracle.envs import OracleVec
from oracle.pixel_preprocessing import PreprocessedVec, noop_count
from pufferlib_b200.environments import ocean, resolve_config
from pufferlib_b200.exceptions import APIUsageError

KINDS = ('pong', 'breakout_pixels')


def tape(kind, h, n, seed):
    k = 6 if kind == 'pong' else 4
    return np.random.default_rng(seed).integers(0, k, size=(h, n)).astype(np.int64)


def plain(kind, n, iparam=()):
    return OracleVec('pong', n, iparam=iparam) if kind == 'pong' else BreakoutPixelsVec(n, iparam=iparam)


@pytest.mark.parametrize('kind', KINDS)
def test_defaults_are_the_plain_oracle(kind):
    """frameskip 1, no no-ops, no episodic life, no clip: every row and info bitwise the plain oracle's."""
    n, h = 3, 150
    iparam = [2, 60] if kind == 'pong' else [40]
    a, b = PreprocessedVec(kind, n, iparam=iparam), plain(kind, n, iparam)
    acts = tape(kind, h, n, 1)
    a.async_reset(5)
    b.async_reset(5)
    ends = 0
    for t in range(h + 1):
        ga, gb = a.recv(), b.recv()
        assert np.array_equal(ga[0], gb[0]), t
        assert np.array_equal(ga[1].view(np.uint32), gb[1].view(np.uint32)) and np.array_equal(ga[2], gb[2]), t
        assert ga[4] == gb[4], t
        ends += len(ga[4])
        if t < h:
            a.send(acts[t])
            b.send(acts[t])
    assert ends > 0


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('skip', [2, 4])
def test_skip_reward_is_the_sum_of_tick_rewards(kind, skip):
    """One env, the action repeated `skip` ticks in the plain oracle: the row reward is the sum of those tick rewards, the
    game ends where the plain game does, and the new frame is the max of the last two tick frames."""
    iparam = [5, 400] if kind == 'pong' else [400]
    a, b = PreprocessedVec(kind, 1, iparam=iparam, frameskip=skip), plain(kind, 1, iparam)
    acts = tape(kind, 300, 1, 7)
    a.async_reset(3)
    b.async_reset(3)
    nonzero = 0
    for t in range(300):
        a.send(acts[t])
        frames, total = [], 0.0
        for _ in range(skip):
            b.send(acts[t])
            o, r, term = b.recv()[:3]
            total += float(r[0])
            frames.append(o[0, 3].copy())
            if term[0]:
                break
        assert a.rewards[0] == np.float32(total) and a.terminals[0] == term[0], t
        want = frames[0] if len(frames) == 1 else np.maximum(frames[-2], frames[-1])
        assert np.array_equal(a.observations[0, 3], want), t
        nonzero += total != 0
        if term[0]:                 # the reset rows: no no-ops, so both are the plain reset row
            b.send(acts[t])
            a.send(acts[t])
            assert np.array_equal(a.observations[0], b.recv()[0][0]) and a.rewards[0] == 0, t
    assert nonzero > 0


@pytest.mark.parametrize('kind', KINDS)
def test_clip_gives_the_signs(kind):
    iparam = [5, 500] if kind == 'pong' else [500]
    a = PreprocessedVec(kind, 8, iparam=iparam, frameskip=4, clip_rewards=True)
    b = PreprocessedVec(kind, 8, iparam=iparam, frameskip=4)
    acts = tape(kind, 500, 8, 2)
    a.async_reset(8)
    b.async_reset(8)
    big = 0
    for t in range(500):
        a.send(acts[t])
        b.send(acts[t])
        assert np.array_equal(a.rewards, np.sign(b.rewards).astype(np.float32)), t
        assert np.array_equal(a.observations, b.observations) and np.array_equal(a.terminals, b.terminals), t
        assert [i['episode_return'] for i in a.infos] == [i['episode_return'] for i in b.infos]   # raw, unclipped
        big += int((np.abs(b.rewards) > 1).sum())
    if kind == 'breakout_pixels':
        assert big > 0, 'no summed brick reward above 1: the clip is not exercised'


def test_life_loss_is_a_terminal_while_the_game_goes_on():
    """episodic_life: a lost life is a terminal row without an info; the next row is a soft reset (all 4 slots one frame,
    reward 0), the game's tick count goes on, and the game's end reports the stats of the whole game."""
    n, h = 4, 1500
    a = PreprocessedVec('breakout_pixels', n, frameskip=4, episodic_life=True)
    b = PreprocessedVec('breakout_pixels', n, frameskip=4)
    acts = tape('breakout_pixels', h, n, 4)
    a.async_reset(1)
    b.async_reset(1)
    lost = games = 0
    for t in range(h):
        was_soft = a.soft.copy()
        a.send(acts[t])
        for e in np.nonzero(was_soft)[0]:
            assert a.rewards[e] == 0 and all(np.array_equal(a.observations[e, k], a.observations[e, 3]) for k in range(3))
        lost += int((a.terminals & ~a.ended).sum())
        games += len(a.infos)
        assert len(a.infos) == int(a.ended.sum())
        for info in a.infos:
            assert info['episode_length'] > 0
    assert lost > 0 and games > 0, (lost, games)
    a.close()
    b.close()


def test_soft_reset_ending_the_game():
    """max_ticks inside a soft reset's no-op step: the row is terminal, reports the game's stats, the next send is a real
    reset."""
    seen = False
    for mt in range(34, 400, 7):       # max_ticks >= 4 * frameskip
        a = PreprocessedVec('breakout_pixels', 1, iparam=[mt], frameskip=8, episodic_life=True)
        a.async_reset(mt)
        acts = tape('breakout_pixels', 200, 1, mt)
        for t in range(200):
            soft = bool(a.soft[0])
            a.send(acts[t])
            if soft and a.terminals[0]:
                assert a.ended[0] and a.rewards[0] == 0
                assert len(a.infos) == 1 and a.infos[0]['episode_length'] == mt
                resets = int(a.resets[0])
                a.send(acts[t])
                assert int(a.resets[0]) == resets + 1 and not a.terminals[0]
                seen = True
                break
        a.close()
        if seen:
            break
    assert seen, 'no game ended inside a soft reset'


@pytest.mark.parametrize('kind', KINDS)
def test_noop_counts(kind):
    """No-op counts lie in [1, noop_max], cover the range, and are reproducible from the seed."""
    iparam = [5, 300] if kind == 'pong' else [300]
    runs = []
    for _ in range(2):
        a = PreprocessedVec(kind, 16, iparam=iparam, noop_max=30, frameskip=4)
        a.async_reset(21)
        acts = tape(kind, 200, 16, 5)
        for t in range(200):
            a.send(acts[t])
        runs.append(list(a.noops))
        a.close()
    assert runs[0] == runs[1]
    counts = [c for _, c in runs[0]]
    assert min(counts) >= 1 and max(counts) <= 30 and len(set(counts)) > 10 and len(counts) > 16
    # the draw is keyed by the global env index: an env at offset 5 draws what env 5 of a vec at offset 0 draws
    b = PreprocessedVec(kind, 1, env_index_offset=5, iparam=iparam, noop_max=30)
    b.async_reset(21)
    assert b.noops[0][1] == noop_count((21 + 5) & ((1 << 64) - 1), 0, 30) == runs[0][5][1]


def test_noop_start_frames_differ():
    a = PreprocessedVec('pong', 8, noop_max=30)
    a.async_reset(3)
    assert len({a.observations[e].tobytes() for e in range(8)}) > 1


# ---- keyword parsing ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', KINDS)
def test_keywords_to_iparam(kind):
    c = ocean.env_creator(kind)
    _, ip, _ = resolve_config(c, [], {})
    assert ip[2:6] == [0, 0, 0, 0]
    kw = {'frameskip': 4, 'noop_max': 30, 'clip_rewards': True}
    if kind == 'breakout_pixels':
        kw['episodic_life'] = True
    _, ip, _ = resolve_config(c, [], kw)
    assert ip[2:6] == [4, 30, int(kind == 'breakout_pixels'), 1]
    _, ip, _ = resolve_config(c, [], {'frameskip': 1, 'noop_max': 0, 'clip_rewards': False})
    assert ip[2:6] == [1, 0, 0, 0]


@pytest.mark.parametrize('kw', [
    {'frameskip': 0}, {'frameskip': 9}, {'frameskip': 2.0}, {'frameskip': True}, {'frameskip': '4'},
    {'noop_max': -1}, {'noop_max': 31}, {'noop_max': 1.5}, {'clip_rewards': 1}, {'clip_rewards': 'yes'},
    {'episodic_life': 1}, {'frame_skip': 4}])
@pytest.mark.parametrize('kind', KINDS)
def test_bad_keywords_refused(kind, kw):
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator(kind), [], kw)


def test_refusals_specific_to_a_kind():
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator('pong'), [], {'episodic_life': True})
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator('pong'), [], {'noop_max': 5, 'max_score': 1})
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator('pong'), [4], {})
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator('breakout_pixels'), [], {'noop_max': 10, 'max_ticks': 10})
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator('pong'), [], {'noop_max': 10, 'max_ticks': 10})
    with pytest.raises(APIUsageError):
        resolve_config(ocean.env_creator('breakout'), [], {'frameskip': 4})
    for kind, mt in (('pong', 'max_ticks'), ('breakout_pixels', 'max_ticks')):     # max_ticks >= 4 * frameskip
        with pytest.raises(APIUsageError):
            resolve_config(ocean.env_creator(kind), [], {'frameskip': 4, mt: 15})
        with pytest.raises(APIUsageError):
            resolve_config(ocean.env_creator(kind), [], {mt: 31, 'frameskip': 8})
        resolve_config(ocean.env_creator(kind), [], {'frameskip': 4, mt: 16})
        resolve_config(ocean.env_creator(kind), [], {'frameskip': 1, mt: 3})
    resolve_config(ocean.env_creator('pong'), [], {'noop_max': 9, 'max_ticks': 10, 'max_score': 2})
