"""pong_versus on the device (PB_ENV_PONG_VERSUS, csrc/env_pong_versus.cu: two agent rows per env, each an (S, 84, 84)
uint8 frame stack from its own side) against the oracle (oracle/pong_versus.py), bit for bit: frames, reward bits,
terminals, truncations, masks and the per-agent infos, at S = 1 and 4, at sizes up to one where every CTA's ring wraps,
and in every vectoriser mode; the per-agent statistics; a captured rollout against the eager one; refusals that launch
nothing; and PPO with Convolutional and LSTMWrapper(Convolutional) on the 2N agent rows."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from oracle.pong_versus import PongVersusVec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.exceptions import APIUsageError
from pufferlib_b200.frameworks import cleanrl

pytestmark = pytest.mark.gpu

FRAME = 84 * 84
GAME = {'max_score': 2, 'max_ticks': 150}


def cpu(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tape(h, n, seed):
    return np.random.default_rng(seed).integers(0, 6, size=(h, 2 * n)).astype(np.int64)


def check_step(t, got, want, infos=True):
    o, r, term, trunc, inf, ids, mask = got
    oo, orr, ot, otr, oinf, oids, om = want
    o = cpu(o)
    assert o.shape == oo.shape, (o.shape, oo.shape)
    if not np.array_equal(o, oo):
        bad = np.nonzero((o != oo).reshape(len(oo), -1).any(1))[0]
        raise AssertionError(f'step {t}: frames differ in rows {bad[:8]} ({len(bad)} rows)')
    assert np.array_equal(cpu(r).view(np.uint32), orr.view(np.uint32)), f'step {t}: reward bits differ'
    assert np.array_equal(cpu(term), ot), f'step {t}: terminals differ'
    assert np.array_equal(cpu(trunc), otr) and np.array_equal(cpu(mask), om), t
    if infos:
        assert inf == oinf, (t, inf[:2], oinf[:2])
        for i in inf:
            assert all(type(v) is int for a in (1, 2) for v in i[a].values()), i


def compare_run(n, h, seed, framestack, game=GAME, offset=0, bound=False, host_buffers=False, infos=True, **make_kw):
    """Device vs oracle on every row of h sends and the reset rows -> (games ended, nonzero rewards, oracle infos)."""
    vec = pvec.make(ocean.env_creator('pong_versus'), env_kwargs={**game, 'framestack': framestack}, num_envs=n,
                    backend=pvec.B200.options(exact_infos=infos, env_index_offset=offset, host_buffers=host_buffers),
                    **make_kw)
    assert vec.num_agents == vec.agents_per_batch == 2 * n and vec.driver_env.num_agents == 2
    assert vec.single_observation_space.shape == (framestack, 84, 84) and vec.obs_bytes == framestack * FRAME
    assert vec.single_action_space.n == 6
    ora = PongVersusVec(n, framestack=framestack, env_index_offset=offset, **game)
    acts = tape(h, n, seed)
    vec.async_reset(seed)
    ora.async_reset(seed)
    exp = None
    if bound:
        exp = clean_pufferl.Experience(2 * n * 8, 4, 2 * n * 8, (framestack, 84, 84), np.uint8, ())
        vec.bind_rollout(exp)
    rewards, all_infos = 0, []
    for t in range(h + 1):
        got = vec.recv()
        want = ora.recv()
        check_step(t, got, want, infos)
        all_infos += want[4]
        rewards += int((want[1] != 0).sum())
        if t < h:
            a = torch.as_tensor(acts[t], device='cuda')
            if bound:
                z = torch.zeros(2 * n, device='cuda')
                exp.store(got[0], z, a, z, got[1], got[2], got[5], got[6])
                if exp.full:
                    exp.sort_training_data()
            vec.send(a if not host_buffers else acts[t])
            ora.send(acts[t])
    stats = vec.episode_stats()
    vec.close()
    ora.close()
    return all_infos, rewards, stats


@pytest.mark.parametrize('framestack', [1, 4])
@pytest.mark.parametrize('n', [1, 5, 33])
def test_vs_oracle(n, framestack):
    infos, rewards, (means, count) = compare_run(n, 400, 3 + n, framestack)
    assert rewards > 0 and len(infos) > 0
    # the per-agent statistics: means over the games ended, of the scores and the game lengths the infos hold
    assert count == len(infos)
    for a in (1, 2):
        assert means[f'{a}/score'] == np.mean([i[a]['score'] for i in infos])
        assert means[f'{a}/episode_length'] == np.mean([i[a]['episode_length'] for i in infos])


@pytest.mark.parametrize('framestack', [1, 4])
def test_every_ring_stage_wraps(framestack):
    """More than 4 x 2 x SMs envs: every CTA's 4-item ring holds two envs and wraps many times per send; short games
    end and reset in the window."""
    n = 4 * 2 * sms() * 3 + 37
    compare_run(n, 40, 5, framestack, game={'max_score': 1, 'max_ticks': 25}, infos=False)


@pytest.mark.parametrize('framestack', [1, 4])
def test_bound_rollout_rows(framestack):
    compare_run(33, 70, 5, framestack, bound=True)


@pytest.mark.parametrize('framestack', [1, 4])
def test_host_buffers(framestack):
    infos, _, _ = compare_run(9, 200, 6, framestack, host_buffers=True)
    assert infos


def test_num_workers_and_env_index_offset():
    """pong_versus keys its draws by global env index, so num_workers keeps one shard; env_index_offset seeds env i as
    the global env offset + i."""
    compare_run(32, 120, 8, 4, num_workers=2)
    compare_run(16, 120, 9, 1, offset=12345)


@pytest.mark.parametrize('groups', [2, 4])
def test_pool_mode(groups):
    """batch_size counts envs: each group returns 2 * batch_size agent rows, round-robin, every env following the
    oracle."""
    n, h = 24, 80
    b = n // groups
    vec = pvec.make(ocean.env_creator('pong_versus'), env_kwargs={**GAME, 'framestack': 4}, num_envs=n,
                    backend=pvec.B200, batch_size=b)
    assert isinstance(vec, pvec.B200Pool) and vec.agents_per_batch == 2 * b and vec.num_agents == 2 * n
    ora = PongVersusVec(n, framestack=4, **GAME)
    acts = tape(h, n, 4)
    vec.async_reset(7)
    ora.async_reset(7)
    for t in range(h):
        oo, orr, ot, _, _, _, _ = ora.recv()
        for g in range(groups):
            o, r, term, _, _, ids, _ = vec.recv()
            lo, hi = 2 * g * b, 2 * (g + 1) * b
            assert np.array_equal(ids, np.arange(lo, hi))
            assert np.array_equal(cpu(o), oo[lo:hi]) and np.array_equal(cpu(r).view(np.uint32), orr[lo:hi].view(np.uint32))
            assert np.array_equal(cpu(term), ot[lo:hi]), (t, g)
            vec.send(torch.as_tensor(acts[t, lo:hi], device='cuda'))
        ora.send(acts[t])
    vec.close()


def test_one_frame_is_the_newest_of_four():
    n, h = 300, 200
    vecs = [pvec.make(ocean.env_creator('pong_versus'), env_kwargs={**GAME, 'framestack': s}, num_envs=n,
                      backend=pvec.B200.options(exact_infos=True)) for s in (1, 4)]
    acts = tape(h, n, 21)
    for v in vecs:
        v.async_reset(21)
    ends = 0
    for t in range(h + 1):
        (o1, r1, d1, _, i1, _, _), (o4, r4, d4, _, i4, _, _) = vecs[0].recv(), vecs[1].recv()
        assert torch.equal(o1, o4[:, 3:]), t
        assert torch.equal(r1.view(torch.int32), r4.view(torch.int32)) and torch.equal(d1, d4) and i1 == i4, t
        ends += len(i1)
        if t < h:
            a = torch.as_tensor(acts[t], device='cuda')
            for v in vecs:
                v.send(a)
    assert ends > 0 and vecs[0].episode_stats() == vecs[1].episode_stats()
    for v in vecs:
        v.close()


@pytest.mark.parametrize('framestack', [1, 4])
def test_captured_rollout_equals_eager(framestack):
    n, h = 64, 40
    acts = torch.as_tensor(tape(h, n, 3), device='cuda')
    opts = {'max_score': 1, 'max_ticks': 30, 'framestack': framestack}

    def run(capture):
        vec = pvec.make(ocean.env_creator('pong_versus'), env_kwargs=opts, num_envs=n, backend=pvec.B200)
        vec.async_reset(11)
        vec.recv()
        vec.send(acts[0])
        vec.recv()
        torch.cuda.synchronize()
        obs = torch.zeros((h, 2 * n, framestack, 84, 84), dtype=torch.uint8, device='cuda')
        rew = torch.zeros((h, 2 * n), device='cuda')
        term = torch.zeros((h, 2 * n), dtype=torch.bool, device='cuda')

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


def test_library_info_and_refusals_launch_nothing():
    L = _native.lib()
    cfg = _native.EnvConfig(kind=_native.ENV_KINDS['pong_versus'], num_envs=3, device=0)
    h = C.c_void_p()
    _native.check(L.pb_env_create(C.byref(cfg), C.byref(h)))
    info, agents = _native.EnvInfo(), C.c_int32()
    _native.check(L.pb_env_get_info(h, C.byref(info)))
    _native.check(L.pb_env_agents_per_env(h, C.byref(agents)))
    assert agents.value == 2 and info.num_actions == 6 and info.obs_bytes == 4 * FRAME and info.obs_ndim == 3
    out = (C.c_double * 4)()
    _native.check(L.pb_env_agent_stats_read(h, out, 1, None))
    assert list(out) == [0.0] * 4
    L.pb_env_destroy(h)
    bad = [(0, 16), (0, -1), (1, 65536), (1, -5), (6, 2), (6, 3), (6, 5), (6, -1), (7, 1)]
    bad += [(k, 1) for k in (2, 3, 4, 5)] + [(2, 4), (3, 30)]
    for k, v in bad:
        ip = [0] * 8
        ip[k] = v
        cfg = _native.EnvConfig(kind=_native.ENV_KINDS['pong_versus'], num_envs=4, device=0, iparam=(C.c_int32 * 8)(*ip))
        h = C.c_void_p()
        l0 = L.pb_launch_count()
        assert L.pb_env_create(C.byref(cfg), C.byref(h)) == _native.PB_ERR_INVALID, (k, v)
        assert L.pb_launch_count() == l0 and not h.value, (k, v)
        assert 'pong_versus' in _native.last_error()
    for kw in ({'frameskip': 4}, {'noop_max': 30}, {'episodic_life': True}, {'clip_rewards': True}, {'framestack': 2},
               {'max_score': 16}, {'max_ticks': 0}):
        l0 = L.pb_launch_count()
        with pytest.raises(APIUsageError):
            pvec.make(ocean.env_creator('pong_versus'), env_kwargs=kw, num_envs=4, backend=pvec.B200)
        assert L.pb_launch_count() == l0, kw


def test_negative_score_sums():
    """The per-agent score sums are signed (two's complement on the device): over games that both seats win, the two
    means are exact negatives."""
    infos, _, (means, count) = compare_run(40, 300, 17, 1, game={'max_score': 1, 'max_ticks': 200})
    assert count == len(infos) > 0
    assert means['1/score'] == -means['2/score']
    assert any(i[1]['score'] < 0 for i in infos) and any(i[1]['score'] > 0 for i in infos)


# ---- PPO on the agent rows --------------------------------------------------------------------------------------------
def plans_of(monkeypatch):
    plans = []
    update_plan = clean_pufferl.update_plan
    monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(update_plan(d)) or plans[-1])
    return plans


def trainer(n, h, bptt, nm, framestack, recurrent):
    from test_gpu_config_updates import ppo_config
    vec = pvec.make(ocean.env_creator('pong_versus'), env_kwargs={'framestack': framestack}, num_envs=n,
                    backend=pvec.B200)
    torch.manual_seed(0)
    if recurrent:
        net = models.LSTMWrapper(vec.driver_env, models.Convolutional(vec.driver_env, framestack=framestack),
                                 input_size=512, hidden_size=512)
        pol = cleanrl.RecurrentPolicy(net, seed=3).cuda()
        cfg = dict(fused_loss=True, learning_rate=2.5e-4, cuda_graph=True)
    else:
        pol = cleanrl.Policy(models.Convolutional(vec.driver_env, framestack=framestack), fused_sample=True,
                             seed=3).cuda()
        cfg = dict(learning_rate=2.5e-4, cuda_graph=True)
    return clean_pufferl.create(ppo_config('pong_versus', 2 * n, h, bptt, nm, **cfg), vec, pol)


@pytest.mark.parametrize('framestack, recurrent, plan', [(4, False, ('model', 'gathered')),
                                                         (1, True, ('cudnn_conv', 'segments'))])
def test_ppo_on_agent_rows(framestack, recurrent, plan, monkeypatch):
    """Convolutional(framestack=4) and LSTMWrapper(Convolutional(framestack=1), 512, 512) at 128 envs (256 agent rows) x
    32 steps: two evaluate() + train() iterations with finite losses, pong's plans, both graphs captured, conv1 on its
    uint8 kernel at S frames and conv2 / conv3 on the TF32 kernels."""
    plans = plans_of(monkeypatch)
    conv1, trunk = [], []
    c1, tr = models._Conv1U8Function.apply, models._ConvReLUTF32Function.apply
    monkeypatch.setattr(models._Conv1U8Function, 'apply', lambda *a: conv1.append(a[0].shape[-3]) or c1(*a))
    monkeypatch.setattr(models._ConvReLUTF32Function, 'apply', lambda *a: trunk.append(a[-1]) or tr(*a))
    data = trainer(128, 32, 8, 2, framestack, recurrent)
    assert data.experience.obs.shape == (256 * 32, framestack, 84, 84)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        losses = [data.losses.policy_loss, data.losses.value_loss, data.losses.entropy]
        assert np.isfinite(losses).all(), losses
    assert (plans[-1].engine, plans[-1].form) == plan, plans[-1]
    assert data.graph_state == 2 and data.train_graph_state == 2, (data.graph_state, data.train_graph_state)
    assert conv1 and set(conv1) == {framestack}
    assert trunk
    clean_pufferl.close(data)
