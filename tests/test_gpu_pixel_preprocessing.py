"""The Atari preprocessing layer of pong and breakout_pixels (frameskip with max-pooling, no-op starts, episodic life,
reward clipping; oracle/SPEC_PIXEL_PREPROCESSING.md) on the device against its oracle (oracle/pixel_preprocessing.py over
the unchanged game oracles): bit-exact frame stacks, reward bits, terminals, truncations, masks and infos, each option
alone and the reference's stack, in every vectoriser mode; refusals; a captured rollout; and training with both graphs
captured."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.exceptions import APIUsageError
from pufferlib_b200.frameworks import cleanrl
from oracle.pixel_preprocessing import PreprocessedVec

pytestmark = pytest.mark.gpu

SHAPE = (4, 84, 84)
# short games, so that game overs, pong points, lost lives and max_ticks all happen within a test's horizon
GAME = {'pong': {'max_score': 2, 'max_ticks': 100}, 'breakout_pixels': {'max_ticks': 300}}
CONFIGS = {
    'skip': {'frameskip': 4},
    'noop': {'noop_max': 30},
    'life': {'episodic_life': True},
    'clip': {'clip_rewards': True},
    'reference': {'frameskip': 4, 'noop_max': 30, 'episodic_life': True, 'clip_rewards': True},
}
CASES = [(k, c) for k in GAME for c in CONFIGS if not (k == 'pong' and c == 'life')]


def opts_of(kind, config):
    o = dict(CONFIGS[config])
    if kind == 'pong':
        o.pop('episodic_life', None)
    return o


def iparam_of(kind, game):
    if kind == 'pong':
        return [game.get('max_score', 0), game.get('max_ticks', 0)]
    return [game.get('max_ticks', 0)]


def cpu(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def tape(kind, h, n, seed):
    if kind == 'pong':
        return np.random.default_rng(seed).integers(0, 6, size=(h, n)).astype(np.int64)
    # FIRE-heavy, so balls launch early, bricks fall and lives are lost
    return np.random.default_rng(seed).choice(4, size=(h, n), p=[0.2, 0.3, 0.25, 0.25]).astype(np.int64)


def oracle(kind, n, opts, game, offset=0):
    return PreprocessedVec(kind, n, env_index_offset=offset, iparam=iparam_of(kind, game), **opts)


def check_step(t, got, want, infos=True):
    o, r, term, trunc, inf, _, mask = got
    oo, orr, ot, _, oinf, _, _ = want
    o = cpu(o)
    if not np.array_equal(o, oo):
        bad = np.nonzero((o != oo).reshape(len(oo), -1).any(1))[0]
        raise AssertionError(f'step {t}: frames differ in envs {bad[:8]} ({len(bad)} envs)')
    assert np.array_equal(cpu(r).view(np.uint32), orr.view(np.uint32)), f'step {t}: reward bits differ'
    assert np.array_equal(cpu(term), ot), f'step {t}: terminals differ'
    assert not cpu(trunc).any() and cpu(mask).all(), t
    if infos:
        assert len(inf) == len(oinf), (t, len(inf), len(oinf))
        for a, b in zip(inf, oinf):
            assert a == b, (t, a, b)


def compare_run(kind, n, h, seed, opts, game=None, offset=0, bound=False, host_buffers=False, infos=True, **make_kw):
    """Device vs oracle, every row of h steps (+ the reset row) -> counts of (game ends, life-loss rows, soft resets that
    ended a game, nonzero rewards)."""
    game = GAME[kind] if game is None else game
    vec = pvec.make(ocean.env_creator(kind), env_kwargs={**game, **opts}, num_envs=n,
                    backend=pvec.B200.options(exact_infos=infos, env_index_offset=offset, host_buffers=host_buffers),
                    **make_kw)
    ora = oracle(kind, n, opts, game, offset)
    acts = tape(kind, h, n, seed)
    vec.async_reset(seed)
    ora.async_reset(seed)
    exp = None
    if bound:
        rows = 8
        exp = clean_pufferl.Experience(n * rows, 4, n * rows, SHAPE, np.uint8, ())
        vec.bind_rollout(exp)
    ends = lost = soft_ends = rewards = 0
    soft = np.zeros(n, dtype=bool)          # a soft reset was pending before the latest send
    for t in range(h + 1):
        got = vec.recv()
        want = ora.recv()
        check_step(t, got, want, infos)
        ends += int(ora.ended.sum())
        lost += int((ora.terminals & ~ora.ended).sum())
        soft_ends += int((soft & ora.ended).sum())
        rewards += int((want[1] != 0).sum())
        if t < h:
            a = torch.as_tensor(acts[t], device='cuda')
            if bound:
                z = torch.zeros(n, device='cuda')
                exp.store(got[0], z, a, z, got[1], got[2], got[5], got[6])
                if exp.full:
                    exp.sort_training_data()
            soft = ora.soft.copy()
            vec.send(a)
            ora.send(acts[t])
    vec.close()
    ora.close()
    return ends, lost, soft_ends, rewards


# ---- 1. device vs oracle: each option alone and the reference's stack ------------------------------------------------
@pytest.mark.parametrize('n', [1, 5, 33, 263])
@pytest.mark.parametrize('kind,config', CASES)
def test_vs_oracle(kind, config, n):
    h = 250 if n <= 33 else 40
    opts = opts_of(kind, config)
    ends, lost, _, rewards = compare_run(kind, n, h, 3 + n, opts)
    ticks = h * opts.get('frameskip', 1)        # breakout: bricks from about tick 60, lost lives from about 140
    if n >= 5 and ticks >= 100:
        assert rewards > 0
    if n >= 5 and ticks > GAME[kind]['max_ticks'] + 30:
        assert ends > 0
    if n >= 5 and ticks >= 250 and 'episodic_life' in opts:
        assert lost > 0


def test_game_ends_inside_a_soft_reset():
    """breakout at max_ticks 150 under the reference stack: many envs lose a life just before tick 150, so the soft reset's
    no-op step runs into max_ticks; those rows are terminal, report the game, and the next send is a real reset."""
    ends, lost, soft_ends, _ = compare_run('breakout_pixels', 33, 120, 7, CONFIGS['reference'], game={'max_ticks': 150})
    assert soft_ends > 0 and lost > 0 and ends > soft_ends, (ends, lost, soft_ends)


def test_clip_applies_to_the_step_sum():
    """breakout at frameskip 8: steps whose ticks hit two bricks sum to 2 or more, and clip to 1 (not to their tick count)."""
    opts = {'frameskip': 8, 'clip_rewards': True}
    ora = oracle('breakout_pixels', 33, {'frameskip': 8}, GAME['breakout_pixels'])
    acts = tape('breakout_pixels', 80, 33, 12)
    ora.async_reset(12)
    sums = []
    for t in range(80):
        ora.send(acts[t])
        sums.append(ora.rewards.copy())
    ora.close()
    assert (np.array(sums) >= 2).sum() > 0
    compare_run('breakout_pixels', 33, 80, 12, opts)


def test_every_ring_stage_wraps():
    """More than 4 x 2 x SMs envs: every CTA runs past its 4-stage ring."""
    n = 4 * 2 * torch.cuda.get_device_properties(0).multi_processor_count + 37
    for kind in GAME:
        opts = opts_of(kind, 'reference')
        compare_run(kind, n, 12, 5, opts, game={'max_ticks': 40} if kind == 'breakout_pixels' else
                    {'max_score': 2, 'max_ticks': 40}, infos=False)


# ---- 2. every vectoriser mode ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', list(GAME))
def test_bound_rollout_rows(kind):
    compare_run(kind, 33, 70, 5, opts_of(kind, 'reference'), bound=True)


@pytest.mark.parametrize('kind', list(GAME))
def test_host_buffers(kind):
    """host_buffers: the info dicts come from the pinned rows and the device's game-ended bytes."""
    ends, _, _, _ = compare_run(kind, 33, 100, 6, opts_of(kind, 'reference'), host_buffers=True)
    assert ends > 0


def test_num_workers():
    compare_run('breakout_pixels', 32, 80, 8, CONFIGS['reference'], num_workers=2)


def test_env_index_offset():
    compare_run('breakout_pixels', 16, 80, 9, CONFIGS['reference'], offset=1000)
    compare_run('pong', 16, 80, 9, opts_of('pong', 'reference'), offset=12345)


@pytest.mark.parametrize('groups', [2, 4])
def test_pool_mode(groups):
    """batch_size < num_envs: groups returned round-robin, every env's rows equal to the oracle's."""
    n, h, kind = 64, 60, 'breakout_pixels'
    b = n // groups
    opts = CONFIGS['reference']
    vec = pvec.make(ocean.env_creator(kind), env_kwargs={**GAME[kind], **opts}, num_envs=n, backend=pvec.B200,
                    batch_size=b)
    assert isinstance(vec, pvec.B200Pool)
    ora = oracle(kind, n, opts, GAME[kind])
    acts = tape(kind, h, n, 4)
    vec.async_reset(7)
    ora.async_reset(7)
    for t in range(h):
        oo, orr, ot, _, _, _, _ = ora.recv()
        for g in range(groups):
            o, r, term, _, _, ids, _ = vec.recv()
            lo, hi = g * b, (g + 1) * b
            assert np.array_equal(ids, np.arange(lo, hi))
            assert np.array_equal(cpu(o), oo[lo:hi]) and np.array_equal(cpu(r), orr[lo:hi]), (t, g)
            assert np.array_equal(cpu(term), ot[lo:hi]), (t, g)
            vec.send(torch.as_tensor(acts[t, lo:hi], device='cuda'))
        ora.send(acts[t])
    vec.close()


# ---- 3. defaults, refusals, capture -----------------------------------------------------------------------------------
def rollout(kind, env_kwargs, n, h, seed):
    vec = pvec.make(ocean.env_creator(kind), env_kwargs=env_kwargs, num_envs=n, backend=pvec.B200.options(exact_infos=True))
    acts = tape(kind, h, n, seed)
    vec.async_reset(seed)
    rows = []
    for t in range(h + 1):
        o, r, term, trunc, inf, _, m = vec.recv()
        rows.append((cpu(o).copy(), cpu(r).copy(), cpu(term).copy(), cpu(trunc).copy(), cpu(m).copy(), inf))
        if t < h:
            vec.send(torch.as_tensor(acts[t], device='cuda'))
    stats = vec.episode_stats()
    vec.close()
    return rows, stats


@pytest.mark.parametrize('kind', list(GAME))
def test_explicit_defaults_equal_no_keywords(kind):
    explicit = {'frameskip': 1, 'noop_max': 0, 'clip_rewards': False}
    if kind == 'breakout_pixels':
        explicit['episodic_life'] = False
    a, sa = rollout(kind, dict(GAME[kind]), 33, 320, 2)      # past max_ticks: games end
    b, sb = rollout(kind, {**GAME[kind], **explicit}, 33, 320, 2)
    assert sa == sb and sa[1] > 0
    for t, (x, y) in enumerate(zip(a, b)):
        for u, v in zip(x[:5], y[:5]):
            assert np.array_equal(u, v), t
        assert x[5] == y[5], t


def test_refusals_launch_nothing():
    lib = _native.lib()
    bad = [('pong', {2: 9}), ('pong', {2: -1}), ('pong', {3: 31}), ('pong', {4: 1}), ('pong', {5: 2}),
           ('pong', {3: 5, 0: 1}), ('pong', {3: 10, 1: 10}), ('breakout_pixels', {3: 20, 0: 20}),
           ('breakout_pixels', {4: 2}), ('breakout_pixels', {2: 100}), ('breakout_pixels', {2: 4, 0: 15}),
           ('pong', {2: 8, 1: 31})]
    for kind, ip in bad:
        iparam = [0] * 8
        for k, v in ip.items():
            iparam[k] = v
        cfg = _native.EnvConfig(kind=_native.ENV_KINDS[kind], num_envs=4, device=0, iparam=(C.c_int32 * 8)(*iparam))
        h = C.c_void_p()
        l0 = lib.pb_launch_count()
        assert lib.pb_env_create(C.byref(cfg), C.byref(h)) == _native.PB_ERR_INVALID, (kind, ip)
        assert lib.pb_launch_count() == l0 and not h.value, (kind, ip)
    for kind, kw in [('pong', {'episodic_life': True}), ('pong', {'frameskip': 0}), ('breakout_pixels', {'noop_max': 31}),
                     ('breakout_pixels', {'clip_rewards': 1}), ('breakout', {'frameskip': 4})]:
        l0 = lib.pb_launch_count()
        with pytest.raises(APIUsageError):
            pvec.make(ocean.env_creator(kind), env_kwargs=kw, num_envs=4, backend=pvec.B200)
        assert lib.pb_launch_count() == l0, (kind, kw)


@pytest.mark.parametrize('kind', list(GAME))
def test_captured_rollout_equals_eager(kind):
    """h sends captured in one CUDA graph and replayed: every row equal to the same sends run eagerly."""
    n, h = 64, 40
    opts = {**GAME[kind], **opts_of(kind, 'reference')}
    acts = torch.as_tensor(tape(kind, h, n, 3), device='cuda')

    def run(capture):
        vec = pvec.make(ocean.env_creator(kind), env_kwargs=opts, num_envs=n, backend=pvec.B200)
        vec.async_reset(11)
        vec.recv()
        vec.send(acts[0])           # the first send checks the actions on the host: not capturable
        vec.recv()
        torch.cuda.synchronize()
        obs = torch.zeros((h, n, *SHAPE), dtype=torch.uint8, device='cuda')
        rew = torch.zeros((h, n), device='cuda')
        term = torch.zeros((h, n), dtype=torch.bool, device='cuda')

        def body():
            for t in range(1, h):
                vec.send(acts[t])
                o, r, d, _, _, _, _ = vec.recv()
                obs[t].copy_(o)
                rew[t].copy_(r)
                term[t].copy_(d)
        if capture:
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                with torch.cuda.graph(g, stream=s):
                    body()
            torch.cuda.current_stream().wait_stream(s)
            g.replay()
        else:
            body()
        torch.cuda.synchronize()
        out = cpu(obs), cpu(rew), cpu(term)
        vec.close()
        return out
    eager, graph = run(False), run(True)
    for x, y in zip(eager, graph):
        assert np.array_equal(x, y)
    assert eager[2].any()


# ---- 4. training with the reference stack -----------------------------------------------------------------------------
def train_run(kind, recurrent, monkeypatch):
    """Four evaluate() + train() iterations at 256 envs x 32 steps with max_ticks 200 (about 50 agent steps a game) -> the
    update engine of every train()."""
    from test_gpu_config_updates import ppo_config
    plans = []
    update_plan = clean_pufferl.update_plan
    monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(update_plan(d)) or plans[-1])
    n, h = 256, 32
    env_kwargs = {**opts_of(kind, 'reference'), 'max_ticks': 200}
    vec = pvec.make(ocean.env_creator(kind), env_kwargs=env_kwargs, num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    if recurrent:
        net = models.LSTMWrapper(vec.driver_env, models.Convolutional(vec.driver_env), input_size=512, hidden_size=512)
        pol = cleanrl.RecurrentPolicy(net, seed=3).cuda()
        cfg = ppo_config(kind, n, h, 8, 2, fused_loss=True, learning_rate=2.5e-4, cuda_graph=True)
    else:
        pol = cleanrl.Policy(models.Convolutional(vec.driver_env, framestack=4, flat_size=3136), fused_sample=True,
                             seed=3).cuda()
        cfg = ppo_config(kind, n, h, 8, 2, learning_rate=2.5e-4, cuda_graph=True)
    data = clean_pufferl.create(cfg, vec, pol)
    seen = False
    for it in range(4):
        stats, _ = clean_pufferl.evaluate(data)
        seen |= 'episode_return' in stats and 'episode_length' in stats
        clean_pufferl.train(data)
        losses = [data.losses.policy_loss, data.losses.value_loss, data.losses.entropy]
        assert all(np.isfinite(x) for x in losses), (it, losses)
    assert data.graph_state == 2 and data.train_graph_state == 2, (data.graph_state, data.train_graph_state)
    assert seen, 'no episode mean reported after the games ended'
    clean_pufferl.close(data)
    return [p.engine for p in plans]


@pytest.mark.parametrize('kind', list(GAME))
def test_convolutional_trains_with_the_reference_stack(kind, monkeypatch):
    train_run(kind, False, monkeypatch)


def test_conv_lstm_trains_with_the_reference_stack(monkeypatch):
    plans = train_run('breakout_pixels', True, monkeypatch)
    assert plans[-1] == 'cudnn_conv', plans
