"""The `framestack` keyword of pong and breakout_pixels (1 or 4 frames per observation row) without a GPU: the keyword's
way to pb_env_config.iparam[6], every refusal, and the one-frame oracle (tests/framestack_oracle.py) against the
four-frame oracles: its frame is the newest slot of theirs, and rewards, terminals, truncations and infos are equal,
across resets, game ends, soft resets and each preprocessing option."""
import numpy as np
import pytest

from pufferlib_b200.environments import ocean, resolve_config
from pufferlib_b200.exceptions import APIUsageError
from oracle.breakout_pixels import BreakoutPixelsVec
from oracle.envs import OracleVec
from oracle.pixel_preprocessing import PreprocessedVec
from framestack_oracle import FrameStackVec

KINDS = ('pong', 'breakout_pixels')
GAME = {'pong': {'max_score': 2, 'max_ticks': 100}, 'breakout_pixels': {'max_ticks': 150}}
CONFIGS = {
    'plain': {},
    'skip': {'frameskip': 4},
    'noop': {'noop_max': 30},
    'life': {'episodic_life': True},
    'clip': {'clip_rewards': True},
    'reference': {'frameskip': 4, 'noop_max': 30, 'episodic_life': True, 'clip_rewards': True},
}
CASES = [(k, c) for k in KINDS for c in CONFIGS if not (k == 'pong' and c == 'life')]


def iparam(kind, **kw):
    return resolve_config(ocean.env_creator(kind), (), kw)[1]


# ---- keyword -> iparam[6] ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', KINDS)
def test_keyword_sets_iparam6(kind):
    assert iparam(kind)[6] == 0
    assert iparam(kind, framestack=4)[6] == 4
    assert iparam(kind, framestack=1)[6] == 1
    assert iparam(kind, framestack=np.int64(1))[6] == 1
    ref = {'frameskip': 4, 'noop_max': 30, 'clip_rewards': True, **({'episodic_life': True} if kind != 'pong' else {})}
    with_opts = iparam(kind, framestack=1, **ref)
    assert with_opts[6] == 1 and with_opts[:6] == iparam(kind, **ref)[:6]


def test_no_keyword_is_todays_iparam():
    assert iparam('pong') == [0] * 8
    assert iparam('breakout_pixels') == [0] * 8
    assert iparam('pong', max_score=3, max_ticks=200) == [3, 200, 0, 0, 0, 0, 0, 0]
    assert iparam('breakout_pixels', max_ticks=500, frameskip=4) == [500, 0, 4, 0, 0, 0, 0, 0]


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('value', [True, False, 1.0, 4.0, '1', '4', None, 0, 2, 3, 5, -1, 8])
def test_bad_values_refused(kind, value):
    with pytest.raises(APIUsageError, match='framestack'):
        iparam(kind, framestack=value)


@pytest.mark.parametrize('kind', ['squared', 'breakout', 'snake', 'memory', 'password', 'stochastic', 'bandit'])
def test_non_pixel_kinds_refuse_the_keyword(kind):
    with pytest.raises(APIUsageError, match='framestack'):
        iparam(kind, framestack=1)


def test_multiagent_refuses_the_keyword():
    with pytest.raises(APIUsageError):
        iparam('multiagent', framestack=1)


# ---- the one-frame oracle against the four-frame oracles ---------------------------------------------------------------
def game_iparam(kind):
    g = GAME[kind]
    return [g['max_score'], g['max_ticks']] if kind == 'pong' else [g['max_ticks']]


def tape(kind, h, n, seed):
    if kind == 'pong':
        return np.random.default_rng(seed).integers(0, 6, size=(h, n)).astype(np.int64)
    return np.random.default_rng(seed).choice(4, size=(h, n), p=[0.2, 0.3, 0.25, 0.25]).astype(np.int64)


def four_frame_oracle(kind, n, opts):
    """The existing oracle of the four-frame env: the plain game oracles for the defaults, else PreprocessedVec."""
    if not opts:
        if kind == 'pong':
            return OracleVec('pong', n, iparam=game_iparam(kind))
        return BreakoutPixelsVec(n, iparam=game_iparam(kind))
    return PreprocessedVec(kind, n, iparam=game_iparam(kind), **opts)


def infos_equal(a, b):
    return len(a) == len(b) and all(x == y for x, y in zip(a, b))


@pytest.mark.parametrize('kind,config', CASES)
def test_one_frame_is_the_newest_slot(kind, config):
    n, h, seed = 6, 260, 4
    opts = dict(CONFIGS[config])
    one = FrameStackVec(kind, n, framestack=1, iparam=game_iparam(kind), **opts)
    four = FrameStackVec(kind, n, framestack=4, iparam=game_iparam(kind), **opts)
    ref = four_frame_oracle(kind, n, opts)
    acts = tape(kind, h, n, seed)
    for o in (one, four, ref):
        o.async_reset(seed)
    ends = resets = softs = 0
    for t in range(h + 1):
        o1, r1, d1, tr1, i1, _, m1 = one.recv()
        o4, r4, d4, tr4, i4, _, m4 = four.recv()
        oo, orr, od, otr, oi, _, om = ref.recv()
        assert o1.shape == (n, 1, 84, 84) and o4.shape == (n, 4, 84, 84)
        assert np.array_equal(o4, oo), t                  # the restated four-frame stack is the existing oracle's
        assert np.array_equal(o1[:, 0], oo[:, 3]), t
        for r in (r1, r4):
            assert np.array_equal(r.view(np.uint32), orr.view(np.uint32)), t
        assert np.array_equal(d1, od) and np.array_equal(d4, od), t
        assert np.array_equal(tr1, otr) and np.array_equal(tr4, otr), t
        assert np.array_equal(m1, om) and np.array_equal(m4, om), t
        assert infos_equal(i1, oi) and infos_equal(i4, oi), (t, i1, oi)
        ends += len(oi)
        softs += int((one.terminals & ~one.ended).sum())
        if t < h:
            resets += int((d1 & ~one.soft).sum())
            for o in (one, four, ref):
                o.send(acts[t])
    for o in (one, four, ref):
        o.close()
    assert ends > 0 and resets > 0, (ends, resets)
    if config in ('life', 'reference') and kind == 'breakout_pixels':
        assert softs > 0


def test_one_frame_rows_of_a_reset_are_the_frame():
    """After async_reset every slot of the four-frame stack holds the same frame, and that frame is the one-frame row."""
    for kind in KINDS:
        one = FrameStackVec(kind, 3, framestack=1, iparam=game_iparam(kind))
        four = FrameStackVec(kind, 3, framestack=4, iparam=game_iparam(kind))
        one.async_reset(9)
        four.async_reset(9)
        for k in range(4):
            assert np.array_equal(four.observations[:, k], one.observations[:, 0])
        assert one.observations.any()
        one.close()
        four.close()
