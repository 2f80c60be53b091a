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
from util_gpu import check_rollout_dump, restated_draw, softmax64, uniforms

pytestmark = pytest.mark.gpu
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def cpu(x):
    return x.detach().cpu().numpy()


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


@pytest.mark.parametrize('n,h,kwargs', [(128, 32, {}), (512, 128, {}), (256, 64, {'max_ticks': 40}),
                                         (512, 64, {'head_bias_shift': 2.0 ** 20})])
def test_fused_rollout_replays_through_oracle(n, h, kwargs):
    """head_bias_shift: every action logit carries the same large offset (the decoder bias + 2^20, ulp 0.125), which
    leaves the policy unchanged; the draw must not depend on how logsumexp rounds there.  The logits are then restated
    as the kernel forms them: the fp32 value of the head product plus the fp32 bias, added in fp32.  Rows whose head
    product rounds across a 0.125 step are the only ones allowed to differ: at most 1e-3 of them."""
    kwargs = dict(kwargs)
    shift = kwargs.pop('head_bias_shift', 0.0)
    data, vec, pol = make(n, h, fused=True, env_kwargs=kwargs)
    with torch.no_grad():
        pol.policy.decoder.bias += shift
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
        prod = hid_t @ w_cat_r.t()
        out = prod + b_cat
        logits, value = out[:, :n_act], out[:, n_act]
        if shift:      # the logits as the kernel forms them: fp32 head product + fp32 bias, added in fp32
            logits32 = prod[:, :n_act].float() + b_cat[:n_act].float()
            logits = logits32.double()
        norm = logits - logits.logsumexp(-1, keepdim=True)
        lp = norm.gather(-1, exp.actions.view(-1, 1)).squeeze(-1)
        if it == 0:      # step 0: hidden layer and head outputs straight from the kernel, within util_gpu.ACC_F32's bound
            with torch.no_grad():
                eh, th, eo, to = check_rollout_dump(dbg_h, dbg_o, exp.obs[:n], model)
            print(f'[rollout n={n} H={h}] step 0: relu(h) max err {eh:.2e} (bound <= {th:.2e}), heads {eo:.2e} '
                  f'(<= {to:.2e})', flush=True)
            assert bool((exp.values[:n] == dbg_o[:, n_act]).all()), 'stored values != the dumped value head'
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
        if shift:      # logprob = z_a - lse with lse in fp32, rounded to the 0.125 grid: restated in fp32
            lp32 = (logits32 - logits32.logsumexp(-1, keepdim=True)).gather(-1, exp.actions.view(-1, 1)).squeeze(-1)
            off = int(((exp.logprobs - lp32).abs() >= 2e-4).sum())
            print(f'[rollout, head bias + 2^20] iteration {it}: {off} of {n * h} logprobs off the fp32 restatement',
                  flush=True)
            assert off <= 1e-3 * n * h, off
        else:
            assert float((exp.logprobs.double() - lp).abs().max()) < 2e-4
        # sampled action = first k with u < cdf_k, u from (seed, step counter, env row): rows where u is not within 1e-4 of
        # a CDF boundary must agree exactly
        probs = softmax64(logits).reshape(h, n, n_act)
        bad = 0
        for t in range(h):
            want, near = restated_draw(probs[t], uniforms(pol._seed, it * h + t, n), 1e-4)
            bad += int(((want != acts[t]) & ~near).sum())
        if shift:
            print(f'[rollout, head bias + 2^20] iteration {it}: {bad} of {n * h} actions off the restated draw', flush=True)
        assert bad <= (1e-3 * n * h if shift else 0), bad
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
