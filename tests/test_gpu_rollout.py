"""The persistent rollout kernel (pb_rollout_breakout_mlp, csrc/env_breakout.cu): H env steps with the policy in the loop
in one launch.  Env rows must replay bit-exactly through the oracle with the actions the kernel sampled (same dynamics,
same bound-rollout row convention, carry-over between rollouts); policy outputs are checked against fp64 torch math on the
stored observations (the encoder product is TF32 on the tensor core), and the sampled actions against the inverse CDF of
the counter-based uniform.  Reference loop: reference clean_pufferl.py:84-124."""
import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
from pufferlib_b200 import clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from oracle.envs import OracleVec

pytestmark = pytest.mark.gpu
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def cpu(x):
    return x.detach().cpu().numpy()


def mix32(x):
    """pb_mix32 (csrc/pb_common.cuh) on a uint64 array."""
    with np.errstate(over='ignore'):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return (x >> np.uint64(32)).astype(np.uint32)


def uniforms(seed, offset, n):
    with np.errstate(over='ignore'):
        key = (np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(offset) * np.uint64(0xD1B54A32D192ED03)
               + np.arange(n, dtype=np.uint64) * np.uint64(0x2545F4914F6CDD1D))
    return (mix32(key) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def make(n, h, fused, env_kwargs=None, graph=False, seed=5):
    vec = pvec.make(ocean.env_creator('breakout'), env_kwargs=env_kwargs or {}, num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=seed).cuda()
    with torch.no_grad():       # non-trivial heads: the default init gives almost uniform policies
        pol.policy.decoder.weight.mul_(40.0)
        pol.policy.value_head.weight.mul_(3.0)
    cfg = pufferlib_b200.namespace(
        seed=1, torch_deterministic=True, env='breakout', batch_size=n * h, bptt_horizon=16, minibatch_size=n * h // 2,
        cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
        update_epochs=1, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01,
        max_grad_norm=0.5, target_kl=None, anneal_lr=False, total_timesteps=10 ** 9, cuda_graph=graph, fused_rollout=fused)
    return clean_pufferl.create(cfg, vec, pol), vec, pol


@pytest.mark.parametrize('n,h,kwargs', [(128, 32, {}), (512, 128, {}), (256, 64, {'max_ticks': 40})])
def test_fused_rollout_replays_through_oracle(n, h, kwargs):
    data, vec, pol = make(n, h, fused=True, env_kwargs=kwargs)
    ora = OracleVec('breakout', n, iparam=[kwargs.get('max_ticks', 0)])
    ora.async_reset(1)
    model = pol.policy
    w_enc, b_enc = model.encoder.weight.detach().double(), model.encoder.bias.detach().double()
    w_cat, b_cat = (t.detach().double() for t in model.head_matrix())
    n_act = 4
    episodes = []
    from pufferlib_b200 import _native
    dbg_h = torch.full((n, 128), float('nan'), device='cuda')
    dbg_o = torch.full((n, 8), float('nan'), device='cuda')
    _native.lib().pb_rollout_debug_buffers(_native.ptr(dbg_h), _native.ptr(dbg_o))
    for it in range(3):          # rollout boundaries: the closing step's outputs are row 0 of the next rollout
        clean_pufferl.evaluate(data)
        _native.lib().pb_rollout_debug_buffers(None, None)
        assert data.fused_rollouts == it + 1
        exp = data.experience
        assert exp.ptr == n * h and data.global_step == (it + 1) * n * h
        acts, obs = cpu(exp.actions).reshape(h, n), cpu(exp.obs).reshape(h, n, 128)
        rew, done = cpu(exp.rewards).reshape(h, n), cpu(exp.dones).reshape(h, n)
        for t in range(h):
            o, r, d, _, infos, _, _ = ora.recv()
            assert np.array_equal(o, obs[t]), (it, t)
            assert np.array_equal(r.view(np.uint32), rew[t].view(np.uint32)), (it, t)
            assert np.array_equal(d.astype(np.float32), done[t]), (it, t)
            episodes += infos
            ora.send(acts[t])
        # policy outputs on the stored observations (W_enc truncated to TF32 by the tensor core; obs exact in TF32)
        w_t = (model.encoder.weight.detach().view(torch.int32) & ~0x1FFF).view(torch.float32).double()
        b_enc = model.encoder.bias.detach().double()          # the parameters move every train() call
        w_cat, b_cat = (t.detach().double() for t in model.head_matrix())
        x = exp.obs.double()
        hid = torch.relu(x @ w_t.t() + b_enc)
        # the head products run on mma.sync: relu(h) truncated to TF32 by the tensor core, W_heads rounded to TF32 (cvt.rna)
        hid_t = (hid.float().view(torch.int32) & ~0x1FFF).view(torch.float32).double()
        w_cat_r = ((w_cat.float().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32).double()
        out = hid_t @ w_cat_r.t() + b_cat
        logits, value = out[:, :n_act], out[:, n_act]
        norm = logits - logits.logsumexp(-1, keepdim=True)
        lp = norm.gather(-1, exp.actions.view(-1, 1)).squeeze(-1)
        if it == 0:      # step 0: hidden layer and head outputs straight from the kernel
            h0 = hid[:n]
            eh = (dbg_h.double() - h0).abs()
            print(f'[diag] hidden step 0: max err {float(eh.max()):.3e}; per 32-col chunk', [f'{float(eh[:, 32*c:32*c+32].max()):.2e}' for c in range(4)],
                  'rows with err>1e-4:', int((eh.max(1).values > 1e-4).sum()), flush=True)
            eo = (dbg_o[:, :5].double() - out[:n, :5]).abs()
            print(f'[diag] head outputs step 0: max err per head {[f"{float(eo[:, a].max()):.2e}" for a in range(5)]}', flush=True)
            print(f'[diag] stored values vs kernel out[4] at step 0: {float((exp.values[:n].double() - dbg_o[:, 4].double()).abs().max()):.3e}', flush=True)
            o_from_h = (dbg_h.view(torch.int32) & ~0x1FFF).view(torch.float32).double() @ w_cat_r.t() + b_cat
            print(f'[diag] heads recomputed from the kernel hidden vs kernel out: {float((dbg_o[:, :5].double() - o_from_h[:, :5]).abs().max()):.3e}', flush=True)
        dv = float((exp.values.double() - value).abs().max())
        if dv >= 2e-4:       # diagnostics: which reference is the kernel closest to?
            for name, w_ in (('exact W', model.encoder.weight.detach().double()), ('truncated W', w_t)):
                for bias_on in (True, False):
                    h_ = torch.relu(x @ w_.t() + (b_enc if bias_on else 0))
                    o_ = h_ @ w_cat.t() + b_cat
                    print(f'[diag] {name}, b_enc {bias_on}: max|dv| {float((exp.values.double() - o_[:, n_act]).abs().max()):.3e} '
                          f'max|dlogit0| -', flush=True)
            print('[diag] b_cat', b_cat.cpu().numpy(), 'values[:4]', exp.values[:4].cpu().numpy(), 'ref', value[:4].cpu().numpy())
        assert dv < 2e-4, dv
        assert float((exp.logprobs.double() - lp).abs().max()) < 2e-4
        # sampled action = first k with u < cdf_k, u from (seed, step counter, env row): rows where u is not within 1e-4 of
        # a CDF boundary must agree exactly
        cdf = norm.exp().cumsum(-1).cpu().numpy().reshape(h, n, n_act)
        bad = 0
        for t in range(h):
            u = uniforms(pol._seed, it * h + t, n).astype(np.float64)
            want = (u[:, None] >= cdf[t]).sum(-1).clip(max=n_act - 1)
            near = (np.abs(u[:, None] - cdf[t]) < 1e-4).any(-1)
            bad += int(((want != acts[t]) & ~near).sum())
        assert bad == 0, bad
        clean_pufferl.train(data)
        assert np.isfinite(data.losses.policy_loss)
    # device-side EpisodeStats of the last rollout vs the oracle's infos for the same steps are covered by the means
    assert int(cpu(data.policy._counter)[0]) == 3 * h
    clean_pufferl.close(data)


def test_fused_rollout_episode_stats_and_graph():
    """Short episodes: auto-resets, EpisodeStats means through the device-side reduction, and the rollout captured in a
    CUDA graph (constant-bank copies + tensor-map parameters replay correctly)."""
    n, h = 256, 64
    data, vec, pol = make(n, h, fused=True, env_kwargs={'max_ticks': 25}, graph=True)
    ora = OracleVec('breakout', n, iparam=[25])
    ora.async_reset(1)
    for it in range(4):
        stats, _ = clean_pufferl.evaluate(data)
        exp = data.experience
        acts, obs = cpu(exp.actions).reshape(h, n), cpu(exp.obs).reshape(h, n, 128)
        eps = []
        for t in range(h):
            o, r, d, _, infos, _, _ = ora.recv()
            assert np.array_equal(o, obs[t]), (it, t)
            ora.send(acts[t])
            eps += ora.infos
        assert len(eps) > 0
        assert np.isclose(stats['episode_return'], np.mean([i['episode_return'] for i in eps]), rtol=1e-9)
        assert np.isclose(stats['episode_length'], np.mean([i['episode_length'] for i in eps]), rtol=1e-9)
        assert np.isclose(stats['score'], np.mean([i['score'] for i in eps]), rtol=1e-6)
        clean_pufferl.train(data)
    assert data.fused_rollouts >= 2 and data.graph_replays >= 2      # eager call + capture, then replays
    clean_pufferl.close(data)


def test_fused_rollout_matches_loop_at_first_step():
    """Same seeds through the per-step kernels (k_breakout + k_policy_mlp_sample): identical first observations, the same
    uniforms, logits equal to TF32 noise -> the first actions agree except where u sits on a CDF boundary."""
    n, h = 1024, 16
    acts = {}
    for fused in (True, False):
        data, vec, pol = make(n, h, fused=fused)
        clean_pufferl.evaluate(data)
        assert (getattr(data, 'fused_rollouts', 0) == 1) == fused
        acts[fused] = cpu(data.experience.actions).reshape(h, n)
        obs0 = cpu(data.experience.obs).reshape(h, n, 128)[0]
        acts[('obs', fused)] = obs0
        clean_pufferl.close(data)
    assert np.array_equal(acts[('obs', True)], acts[('obs', False)])
    assert np.mean(acts[True][0] == acts[False][0]) > 0.99
