"""pong_versus on the CPU: the oracle (oracle/pong_versus.py over oracle/csrc/pong_versus.c) against the properties
oracle/SPEC_PONG_VERSUS.md states -- zero-sum rewards, the mirror / value-swap identity of the two agents' frames, shared
done flags, per-agent infos whose scores are the agents' returns -- over many seeds and random action tapes, across
resets, game ends and max_ticks, at S = 1 and 4; and the creator's refusals, raised before any device work.  No GPU."""
import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from oracle.pong_versus import PongVersusVec
from pufferlib_b200.environments import ocean, resolve_config
from pufferlib_b200.exceptions import APIUsageError


def swap_mirror(frames):
    """The other agent's view of a frame stack: columns mirrored, paddle values 128 and 192 exchanged."""
    m = frames[..., ::-1].copy()
    p128, p192 = m == 128, m == 192
    m[p128], m[p192] = 192, 128
    return m


def run(n, steps, seed, framestack, max_score=0, max_ticks=0, offset=0, tape_seed=0):
    """Drive the oracle with a random action tape, checking every recv; returns (obs, rewards, terminals, infos) per
    step."""
    rng = np.random.default_rng(tape_seed)
    vec = PongVersusVec(n, framestack=framestack, env_index_offset=offset, max_score=max_score, max_ticks=max_ticks)
    vec.async_reset(seed)
    ret = np.zeros(2 * n)
    length = np.zeros(n, dtype=np.int64)
    reset_next = np.ones(n, dtype=bool)        # the rows async_reset wrote are reset rows
    hist = []
    games = 0
    for t in range(steps):
        o, r, term, trunc, infos, ids, masks = vec.recv()
        assert o.shape == (2 * n, framestack, 84, 84) and o.dtype == np.uint8
        assert np.array_equal(ids, np.arange(2 * n)) and masks.all() and not trunc.any()
        # zero-sum rewards, +0.0 where agent 0's is 0; one done flag per env
        assert np.array_equal(r[1::2], -r[0::2]) and not np.signbit(r[1::2][r[0::2] == 0]).any()
        assert np.isin(r, (-1.0, 0.0, 1.0)).all()
        assert np.array_equal(term[0::2], term[1::2])
        # agent 1's frames are agent 0's seen from the left
        assert np.array_equal(o[1::2], swap_mirror(o[0::2]))
        # each agent's own paddle is 192 on the right, the other's 128 on the left, 24 pixels each unless the ball hides
        # some; a reset row stacks one frame
        assert (o[:, :, :, 4:6] != 192).all() and (o[:, :, :, 78:80] != 128).all()
        if framestack == 4:
            for e in np.nonzero(reset_next)[0]:
                assert (o[2 * e:2 * e + 2] == o[2 * e:2 * e + 2, :1]).all()
        # returns and lengths since the last reset; infos where a game ended, in env order
        ended = np.nonzero(term[0::2])[0]
        ret[~np.repeat(reset_next, 2)] += r[~np.repeat(reset_next, 2)]
        length[~reset_next] += 1
        if t > 0:
            assert len(infos) == len(ended)
            for e, info in zip(ended, infos):
                assert set(info) == {1, 2}
                assert info[1]['score'] == ret[2 * e] and info[2]['score'] == ret[2 * e + 1] == -info[1]['score']
                assert info[1]['episode_length'] == info[2]['episode_length'] == length[e]
                assert max_ticks == 0 or length[e] <= max_ticks
            games += len(ended)
        ret[np.repeat(reset_next, 2)] = 0
        length[reset_next] = 0
        hist.append((o.copy(), r.copy(), term.copy(), [dict(i) for i in infos]))
        reset_next = term[0::2].copy()
        vec.send(rng.integers(0, 6, 2 * n))
    vec.close()
    return hist, games


@pytest.mark.parametrize('framestack', [1, 4])
@pytest.mark.parametrize('seed', [0, 7, 123456789, 2 ** 64 - 3])
def test_oracle_properties_over_seeds(framestack, seed):
    """Short games (max_score 2) end and reset many times within the tape; every recv satisfies the spec's identities."""
    _, games = run(6, 400, seed, framestack, max_score=2, tape_seed=seed % 1000)
    assert games >= 6


@pytest.mark.parametrize('framestack', [1, 4])
def test_oracle_max_ticks_ends_games(framestack):
    """max_ticks ends every game that no one wins first, at exactly max_ticks steps."""
    hist, games = run(4, 200, 3, framestack, max_score=15, max_ticks=17, tape_seed=5)
    lengths = [i[1]['episode_length'] for _, _, _, infos in hist for i in infos]
    assert games == len(lengths) > 0 and max(lengths) == 17


def test_oracle_one_frame_is_newest_of_four():
    """S = 1 rows are the newest slot of the S = 4 rows under the same seed and tape; rewards, flags and infos agree."""
    a, _ = run(5, 300, 11, 1, max_score=2, tape_seed=2)
    b, _ = run(5, 300, 11, 4, max_score=2, tape_seed=2)
    for (o1, r1, t1, i1), (o4, r4, t4, i4) in zip(a, b):
        assert np.array_equal(o1[:, 0], o4[:, 3])
        assert np.array_equal(r1, r4) and np.array_equal(t1, t4) and i1 == i4


def test_oracle_seeds_by_global_env_index():
    """env_index_offset: env i of a shard with offset k plays what env k + i of one big vectoriser plays."""
    n, k = 6, 2
    full = PongVersusVec(n, framestack=1, max_score=2)
    part = PongVersusVec(n - k, framestack=1, env_index_offset=k, max_score=2)
    full.async_reset(9)
    part.async_reset(9)
    rng = np.random.default_rng(4)
    for _ in range(120):
        assert np.array_equal(full.observations[2 * k:], part.observations)
        assert np.array_equal(full.rewards[2 * k:], part.rewards) and np.array_equal(full.terminals[2 * k:], part.terminals)
        a = rng.integers(0, 6, 2 * n)
        full.send(a)
        part.send(a[2 * k:])


def test_oracle_serve_frame():
    """The first frame: both paddles at y = 36..47, the ball at (41, 41) for agent 0 and at columns 41..42 mirrored
    (41..42 again) for agent 1."""
    vec = PongVersusVec(1, framestack=1)
    vec.async_reset(0)
    f0, f1 = vec.observations[0, 0], vec.observations[1, 0]
    for f in (f0, f1):
        assert (f[36:48, 4:6] == 128).all() and (f[36:48, 78:80] == 192).all() and (f[41:43, 41:43] == 255).all()
        assert np.count_nonzero(f) == 24 + 24 + 4


def test_creator_keywords():
    """The creator takes max_score, max_ticks and framestack as keywords; defaults are pong's."""
    c = ocean.env_creator('pong_versus')
    assert c.__name__ == 'make_pong_versus' and c.b200_kind == 'pong_versus'
    assert resolve_config(c, [], {}) == ('pong_versus', [0] * 8, [])
    assert resolve_config(c, [], {'max_score': 3, 'max_ticks': 900, 'framestack': 1}) == \
        ('pong_versus', [3, 900, 0, 0, 0, 0, 1, 0], [])
    assert resolve_config(c, [], {'framestack': 4})[1][6] == 4


@pytest.mark.parametrize('kwargs', [
    {'frameskip': 4}, {'frameskip': 1}, {'noop_max': 30}, {'noop_max': 0}, {'episodic_life': False},
    {'clip_rewards': True}, {'clip_rewards': False},
    {'framestack': 0}, {'framestack': 2}, {'framestack': 3}, {'framestack': 5}, {'framestack': True},
    {'framestack': 4.0}, {'framestack': '4'},
    {'max_score': 0}, {'max_score': 16}, {'max_score': -1}, {'max_score': 2.5}, {'max_score': None},
    {'max_ticks': 0}, {'max_ticks': 65536}, {'max_ticks': '100'},
    {'num_agents': 2}, {'seed': 1},
])
def test_creator_refusals(kwargs):
    """The preprocessing options, a bad framestack / max_score / max_ticks and unknown keywords raise APIUsageError in
    resolve_config, and so in vector.make before any device is touched (no CUDA device needed to see them)."""
    c = ocean.env_creator('pong_versus')
    with pytest.raises(APIUsageError):
        resolve_config(c, [], kwargs)
    with pytest.raises(APIUsageError):
        pvec.make(c, env_kwargs=kwargs, num_envs=2, backend=pvec.B200)


def test_creator_refuses_positional_args():
    c = ocean.env_creator('pong_versus')
    with pytest.raises(APIUsageError):
        resolve_config(c, [5], {})


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the CPU-only path')
def test_valid_config_needs_a_device():
    """A valid config gets as far as the device check: no CPU fallback."""
    with pytest.raises(RuntimeError):
        pvec.make(ocean.env_creator('pong_versus'), num_envs=2, backend=pvec.B200)
