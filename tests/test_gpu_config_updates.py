"""The updates of BASELINE.json's C3 (snake, models.Default on 16 x 16 uint8 observations) and C4 (pong, models.Convolutional)
against fp64, at the shapes those configs run.

1. _DefaultMLPUpdate's hand-written kernel chain on uint8 slab minibatches, stage by stage: the slab view train() hands it
   (Experience.slab_obs), x.float(), one encoder GEMM per slab, the head GEMM, pb_ppo_loss, pb_mlp_tail_backward_ex and the
   slab form of models._gemm_tn.  The encoder weights and bias lie on the 2^-8 grid with |w| <= 0.25 and x is a byte, so
   every product is exact in TF32 and fp32 and every partial sum is a multiple of 2^-8 below 2^15: exact in any order.
   The hidden layer is then known bit for bit, no ReLU mask can differ, and each later stage is checked from the kernel's
   own previous one.  Every row of the rollout buffer outside the minibatch holds byte 255, so a misread slab moves every
   gradient.  Up to C3 itself: G = 4 slabs of R = 1 048 576 rows, M = 4 194 304.
2. train() on snake replayed minibatch by minibatch (the 'slabs' form, the chain), and pb_adv_norm at C3's size.
3. C4: train() with the fused loss ('model' engine) against the policy's forward + the reference loss, the TMA path of
   pb_minibatch_gather against a numpy gather, and train()'s b_obs against the oracle's flatten_batch.

The maxima observed on an H100 80GB HBM3 at a 700 W power limit (one run; the file takes 22 s) are in the docstrings
below and in DESIGN.md §4.
"""
import time
import types

import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from oracle import experience as oexp
from oracle import gae as ogae
from test_gpu_policy_lstm import fake_env
from test_gpu_ppo_loss import reference_loss
from util_gpu import ACC_F32
from util_update import check, claim, clip_offsets, rel

pytestmark = pytest.mark.gpu

LOSS = dict(clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)    # the benchmark's
CHUNK = 1 << 18            # rows per chunk of the fp64 reference: a C3 minibatch in fp64 would be ~9 GB of input alone

# Rounding model of the chain's head GEMM (torch.addmm under TF32).  The library reads each fp32 operand as TF32,
# truncated or rounded to nearest: relative error below 2^-10 either way, so a product of two operands is within
# TF32_PROD = 2^-9 + 2^-20 of the exact product, and is itself exact in fp32 (11 x 11 significant bits).  The K = 128
# products and the bias are then summed in fp32 in whatever order the kernel chooses, which util_gpu.ACC_F32 bounds by
# ACC_F32 times the sum of the addends' magnitudes, at most (1 + TF32_PROD) * S with S = sum_k |h_k w_k| + |b|.  So
#     |out_kernel - out_fp64| <= HEADS_TF32 * S,   HEADS_TF32 = TF32_PROD + (1 + TF32_PROD) * ACC_F32.
# A library kernel that multiplies in fp32 instead stays inside the same bound.
TF32_PROD = 2.0 ** -9 + 2.0 ** -20
HEADS_TF32 = TF32_PROD + (1 + TF32_PROD) * ACC_F32


def cpu(x):
    return x.detach().cpu().numpy()


class MaxRel:
    """max |a - b| over chunks, relative to max |b| over chunks."""

    def __init__(self):
        self.err = self.ref = 0.0

    def add(self, a, b):
        e = float((a.double() - b.double()).abs().max())
        self.err = max(self.err, e if e == e else float('inf'))          # a NaN the kernel left fails the check
        self.ref = max(self.ref, float(b.double().abs().max()))

    @property
    def rel(self):
        return self.err / (self.ref + 1e-30)


# ---- 1. the hand-written chain on uint8 slab minibatches -----------------------------------------------------------------
def make_update(n_act, seed):
    """models.Default on snake's observations with exact-encoder weights, and its _DefaultMLPUpdate."""
    torch.manual_seed(seed)
    pol = cleanrl.Policy(models.Default(fake_env((16, 16), n_act, np.uint8))).cuda()
    m = pol.policy
    with torch.no_grad():
        m.encoder.weight.copy_(torch.randint(-64, 65, m.encoder.weight.shape, device='cuda') / 256.0)
        m.encoder.bias.copy_(torch.randint(-64, 65, m.encoder.bias.shape, device='cuda') / 256.0)
        # the hidden units are of order 300 (x up to 255): heads that give logits and a value of order 1
        for p in (m.decoder.weight, m.value_head.weight):
            p.copy_(torch.randn_like(p) * 4e-4)
        for p in (m.decoder.bias, m.value_head.bias):
            p.copy_(torch.randn_like(p) * 0.1)
    opt = torch.optim.Adam(pol.parameters(), lr=1e-3, eps=1e-5, fused=True)
    manual = clean_pufferl._DefaultMLPUpdate(pufferlib_b200.namespace(policy=pol, optimizer=opt,
                                                                      config=pufferlib_b200.namespace(**LOSS)))
    manual.pack_heads()
    return m, manual


def chain_case(n_act, g_, n_envs, bptt, nm, mb, seed):
    """Minibatch mb of a rollout of n_envs x (G * nm * bptt) uint8 rows in the slab form (G slabs of R = bptt * n_envs
    rows), through _DefaultMLPUpdate.forward_backward, checked stage by stage against fp64.  -> dict of observed errors."""
    dev = torch.device('cuda')
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    model, manual = make_update(n_act, seed)
    cfg = pufferlib_b200.namespace(**LOSS)
    r_, horizon = n_envs * bptt, g_ * nm * bptt
    m = g_ * r_
    buf = torch.full((n_envs * horizon, 16, 16), 255, dtype=torch.uint8, device=dev)
    layout = types.SimpleNamespace(obs=buf, num_envs=n_envs, horizon=horizon, num_minibatches=nm, bptt_horizon=bptt,
                                   obs_shape=(16, 16))
    obs = clean_pufferl.Experience.slab_obs(layout, mb)                  # the view train() hands the chain
    assert obs.shape == (g_, r_, 16, 16) and obs.data_ptr() == buf.data_ptr() + mb * r_ * 256
    for g in range(g_):
        obs[g].copy_(torch.randint(0, 256, (r_, 16, 16), dtype=torch.uint8, device=dev))

    def chunks():              # (first row, last row + 1, x [n, 256] uint8) in slab-major minibatch order
        for g in range(g_):
            for lo in range(0, r_, CHUNK):
                hi = min(lo + CHUNK, r_)
                yield g * r_ + lo, g * r_ + hi, obs[g, lo:hi].reshape(hi - lo, 256)

    w_enc, b_enc = model.encoder.weight.double(), model.encoder.bias.double()
    w_cat, b_cat = manual.w_cat.double(), manual.b_cat.double()
    # old log-probabilities and old values relative to the fp64 policy, returns away from the value-clip midpoint
    # (util_update._case): no row lies within 0.1 * clip of a branch edge of the loss
    act = torch.randint(0, n_act, (m,), device=dev)
    nl64 = torch.empty(m, dtype=torch.float64, device=dev)
    v64 = torch.empty(m, dtype=torch.float64, device=dev)
    with torch.no_grad():
        for lo, hi, x in chunks():
            o = torch.relu(x.double() @ w_enc.t() + b_enc) @ w_cat.t() + b_cat
            nl64[lo:hi] = torch.log_softmax(o[:, :n_act], 1).gather(1, act[lo:hi, None])[:, 0]
            v64[lo:hi] = o[:, n_act]
    olp = (nl64 - torch.log1p(cfg.clip_coef * clip_offsets(m, dev))).float()
    oval = (v64 + cfg.vf_clip_coef * clip_offsets(m, dev)).float()
    adv = torch.randn(m, device=dev)
    # returns above the values on average, as early in training (snake's first value loss is ~16): db_val, the value
    # gradient summed over the rows, is then not a near-cancelling sum whose size says nothing about its rounding
    ret = (v64 + 1.0 + 0.5 * torch.randn(m, dtype=torch.float64, device=dev)).float()
    mid = (v64 + oval.double() + torch.clamp(v64 - oval.double(), -cfg.vf_clip_coef, cfg.vf_clip_coef)) / 2
    gap = ret.double() - mid
    ret += torch.where(gap.abs() < 0.05, torch.where(gap < 0, -0.05, 0.05) - gap, torch.zeros_like(gap)).float()
    del nl64, v64, mid, gap

    batch = pufferlib_b200.namespace(obs=obs, slab_form=True, actions=act, logprobs=olp, values=oval, advantages=adv,
                                     returns=ret, row_slab_stride=None, adv_norm=None)
    assert not manual._fused_ok(obs.flatten(2), cfg), 'uint8 observations take the chain'
    manual._buffers(m)
    for t in (manual.hidden, manual.out, manual.dout, manual.dpre, manual.gflat):
        t.fill_(float('nan'))                 # every element the chain does not write stays NaN
    manual.forward_backward(0, 1, batch, cfg)
    torch.cuda.synchronize()
    print(f'case G={g_} R={r_} M={m} n_act={n_act} nm={nm} mb={mb}', flush=True)

    # the fp64 reference, chunk by chunk: each chunk's loss enters with weight n / M, so the gradients and the statistics
    # add up to those of the whole minibatch
    leaves = [p.detach().double().clone().requires_grad_(True) for p in
              (model.encoder.weight, model.encoder.bias, model.decoder.weight, model.decoder.bias, model.value_head.weight,
               model.value_head.bias)]
    we, be, wd, bd, wv, bv = leaves
    st_ref = torch.zeros(6, dtype=torch.float64, device=dev)
    clipped_ref, hidden_off, out_over, out_err, out_ratio = 0, 0, 0, 0.0, 0.0
    e_dout, e_dpre = MaxRel(), MaxRel()
    hr = manual.head_rows
    tail_ref = [torch.zeros(hr, 128, dtype=torch.float64, device=dev), torch.zeros(hr, dtype=torch.float64, device=dev),
                torch.zeros(128, dtype=torch.float64, device=dev)]
    for lo, hi, x in chunks():
        n, w = hi - lo, (hi - lo) / m
        rows = slice(lo, hi)
        a_, olp_, adv_, ret_, oval_ = (act[rows], olp[rows].double(), adv[rows].double(), ret[rows].double(),
                                       oval[rows].double())
        with torch.enable_grad():
            hid = torch.relu(x.double() @ we.t() + be)
            loss, st = reference_loss(hid @ wd.t() + bd, hid @ wv.t() + bv, a_, olp_, adv_, ret_, oval_, cfg)
            (loss * w).backward()
        st_ref += st * w
        clipped_ref += round(float(st[5]) * n)
        # hidden: the exact value, bit for bit
        kh = manual.hidden[rows]
        hidden_off += int((kh != hid.detach().float()).sum())
        # out: the head GEMM from the kernel's own hidden, within the TF32 bound
        ko, hk = manual.out[rows].double(), kh.double()
        err = (ko - (hk @ w_cat.t() + b_cat)).abs()
        bound = HEADS_TF32 * (hk.abs() @ w_cat.abs().t() + b_cat.abs())
        out_over += int((~(err <= bound)).sum())          # the zero padding columns must be exactly 0; NaN counts
        out_err = max(out_err, float(err.max()))
        out_ratio = max(out_ratio, float((err / bound)[:, :n_act + 1].max()))
        # dOut: fp64 autograd of the loss on the kernel's own out
        lg = ko[:, :n_act].clone().requires_grad_(True)
        vl = ko[:, n_act:n_act + 1].clone().requires_grad_(True)
        with torch.enable_grad():
            (reference_loss(lg, vl, a_, olp_, adv_, ret_, oval_, cfg)[0] * w).backward()
        ref_dout = torch.zeros(n, manual.head_rows, dtype=torch.float64, device=dev)
        ref_dout[:, :n_act], ref_dout[:, n_act] = lg.grad, vl.grad[:, 0]
        e_dout.add(manual.dout[rows], ref_dout)
        # dPre from the kernel's own dOut and hidden
        e_dpre.add(manual.dpre[rows], (manual.dout[rows].double() @ w_cat) * (kh > 0))
        # the tail backward's sums over the rows, from the kernel's own dOut, hidden and dPre
        kd = manual.dout[rows].double()
        tail_ref[0] += kd.t() @ hk
        tail_ref[1] += kd.sum(0)
        tail_ref[2] += manual.dpre[rows].double().sum(0)
    torch.cuda.synchronize()

    errs = {}
    ok = claim(f'hidden bitwise equal to fp64 ({hidden_off} elements differ)', hidden_off == 0)
    ok &= claim(f'out within HEADS_TF32 bound (max err {out_err:.2e}, {out_ratio:.3f} of bound)', out_over == 0)
    errs['out'] = out_err
    errs['dout'], errs['dpre'] = e_dout.rel, e_dpre.rel
    ok &= claim(f'dOut vs fp64 autograd on the kernel out: {e_dout.rel:.3e}', e_dout.rel <= 1e-5)
    ok &= claim(f'dPre vs (dOut W_cat) * (hidden > 0): {e_dpre.rel:.3e}', e_dpre.rel <= 1e-6)
    # pb_mlp_tail_backward_ex's row sums (fp32, 512-row CTAs, then k_reduce_partials) against fp64 sums of the kernel's own
    # rows, 1e-5 of each maximum (the tail-backward precedent): tight enough that one CTA's partial left out of the 8 192 of
    # C3 is seen, which the fp64-autograd bound below is not
    dw_heads, db_heads, db_enc = (manual.tail[:hr * 128].view(hr, 128), manual.tail[(hr + 1) * 128:],
                                  manual.tail[hr * 128:(hr + 1) * 128])
    for name, v, r in zip(('dW_heads', 'db_heads', 'db_enc'), (dw_heads, db_heads, db_enc), tail_ref):
        errs['tail ' + name] = rel(v, r)
        ok &= check(f'{name} vs fp64 sums of the kernel rows', v, r, 1e-5)
    for name, v, r in zip(('W_enc', 'b_enc', 'W_dec', 'b_dec', 'w_val', 'b_val'), manual._keep[1], [p.grad for p in leaves]):
        errs[name] = rel(v, r)
        ok &= check(f'd{name} vs fp64 autograd', v, r, 5e-3)
    ok &= claim('padding rows of dW_heads / db_heads exactly 0',
                bool((dw_heads[n_act + 1:] == 0).all()) and bool((db_heads[n_act + 1:] == 0).all()))
    stats = manual.stats[0]
    st = stats[:6] / m
    st[1] *= 0.5                       # the kernel sums (v - ret)^2; the loss is half its mean
    errs['stats'] = rel(st, st_ref)
    ok &= check('loss statistics vs fp64', st, st_ref, 2e-3)
    clipfrac = clipped_ref / m
    ok &= claim(f'rows on both sides of the clip range (clipfrac {clipfrac:.3f})', 0.2 < clipfrac < 0.8)
    ok &= claim(f'clipped rows {round(float(stats[5]))} == fp64 {clipped_ref}', round(float(stats[5])) == clipped_ref)
    peak = torch.cuda.max_memory_allocated()
    print(f'    peak memory {peak / 2 ** 30:.2f} GiB, {time.perf_counter() - t0:.1f} s', flush=True)
    assert ok, errs
    return errs, peak


# (G, n_envs, bptt, nm, mb): R = 16 * 37 = 592 is ragged against the tail backward's 512-row CTAs and 32-row TMA chunks
SMALL = [(g, ne, 16, 2, 1) for g in (1, 2, 4) for ne in (37, 2048)]


@pytest.mark.parametrize('n_act', [1, 4, 7])
@pytest.mark.parametrize('g_,n_envs,bptt,nm,mb', SMALL, ids=[f'G{s[0]}_R{16 * s[1]}' for s in SMALL])
def test_chain_uint8_slabs_vs_fp64(g_, n_envs, bptt, nm, mb, n_act):
    """G in {1, 2, 4} x R in {592, 32 768} x 1, 4, 7 actions.  Observed over these and the two one-slab cases: hidden
    bitwise; out 1.95e-3 absolute, 0.13 of the HEADS_TF32 bound; dOut 4.2e-7; dPre 1.5e-7; the tail backward's sums
    1.0e-7; the six gradients 6.8e-4 of their maximum (bound 5e-3); loss statistics 4.0e-4 (bound 2e-3); clipfrac 0.48
    to 0.52."""
    chain_case(n_act, g_, n_envs, bptt, nm, mb, seed=g_ * 1000 + n_envs + n_act)


@pytest.mark.parametrize('n_envs,bptt', [(8192, 16), (5461, 3)], ids=['M131072_split', 'M16383_plain'])
def test_chain_one_slab_gemm_forms_vs_fp64(n_envs, bptt):
    """G = 1 at M = 131 072, where the slab form of _gemm_tn splits K into 64 batched slices, and at M = 16 383 (odd),
    where it takes one slice: the plain product."""
    chain_case(4, 1, n_envs, bptt, 2, 1, seed=n_envs)
    assert models._slab_split(1, n_envs * bptt) == (64 if n_envs * bptt == 131072 else 1)


def test_chain_c3_minibatch_vs_fp64():
    """C3 itself: 65 536 envs x 256 steps, bptt 16, 4 minibatches -> minibatch 2 is G = 4 slabs of R = 1 048 576 rows
    (M = 4 194 304) of a 16.7 M-row buffer.  Observed: out 1.83e-3 absolute (0.16 of the bound), dOut 3.4e-7, dPre
    9.8e-8, tail sums 1.9e-7, gradients 5.0e-4 of their maximum, loss statistics 2.3e-4, clipped rows equal; peak memory
    12.5 GiB."""
    errs, peak = chain_case(4, 4, 65536, 16, 4, 2, seed=3)
    assert peak < 20 * 2 ** 30, f'peak memory {peak / 2 ** 30:.1f} GiB'


# ---- 2. train() on snake, replayed --------------------------------------------------------------------------------------
def ppo_config(env, n, h, bptt, nm, **kw):
    cfg = dict(seed=1, torch_deterministic=True, env=env, batch_size=n * h, bptt_horizon=bptt, minibatch_size=n * h // nm,
               cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
               update_epochs=2, norm_adv=True, max_grad_norm=0.5, target_kl=None, anneal_lr=False,
               total_timesteps=10 ** 10, **LOSS)
    cfg.update(kw)
    return pufferlib_b200.namespace(**cfg)


def pack_heads(params, w_cat, b_cat):
    n_act = params[2].shape[0]
    _native.check(_native.lib().pb_pack_heads(_native.ptr(params[2]), _native.ptr(params[3]), _native.ptr(params[4]),
                                              _native.ptr(params[5]), n_act, 128, _native.ptr(w_cat), _native.ptr(b_cat),
                                              None, None, 0, _native.stream_ptr()))


def test_snake_train_slabs_replays_through_gathered_minibatches():
    """train() on snake (2 048 envs x 256 steps, bptt 16, 4 minibatches, 2 epochs, annealed lr, every step clipped) runs
    the chain on slab views of the rollout buffer.  Replayed from a snapshot of the rollout, the parameters and the Adam
    state: minibatch membership and advantages from the oracles in fp64 (compute_gae_f64), the normalisation of
    clean_pufferl.py:211-213 in fp64, each minibatch as contiguous gathered uint8 rows (G = 1) through a second
    _DefaultMLPUpdate on copies of the parameters, then its optimizer_step.  Then pb_adv_norm at C3's size: nm = 4
    slab-major minibatches of 4 194 304 rows against fp64.  Observed: parameters 5.6e-9 apart (bound 1e-3 lr per step),
    Adam moments 5.3e-7 relative, policy loss 1.3e-8, pb_adv_norm 5.5e-7 (bound 2e-6)."""
    n, h, bptt, nm = 2048, 256, 16, 4
    dev = torch.device('cuda')
    vec = pvec.make(ocean.env_creator('snake'), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=3).cuda()
    cfg = ppo_config('snake', n, h, bptt, nm, anneal_lr=True, total_timesteps=4 * n * h, max_grad_norm=1e-3)
    data = clean_pufferl.create(cfg, vec, pol)
    clean_pufferl.evaluate(data)
    clean_pufferl.train(data)                    # the Adam state exists and the learning rate is annealed once
    assert data.train_minibatch_path == 'slabs' and data.manual_update.used_fused is False
    clean_pufferl.evaluate(data)
    exp, model, opt = data.experience, pol.policy, data.optimizer
    params = [model.encoder.weight, model.encoder.bias, model.decoder.weight, model.decoder.bias, model.value_head.weight,
              model.value_head.bias]
    st = [{k: opt.state[p][k].clone() for k in ('exp_avg', 'exp_avg_sq', 'step')} for p in params]
    lr = float(opt.param_groups[0]['lr'])
    assert lr < cfg.learning_rate
    # the replay's model: copies of the parameters and of the Adam state
    n_act = model.decoder.weight.shape[0]
    pol2 = cleanrl.Policy(models.Default(fake_env((16, 16), n_act, np.uint8))).cuda()
    mine = list(pol2.parameters())
    with torch.no_grad():
        for p, q in zip(mine, params):
            p.copy_(q)
    opt2 = torch.optim.Adam(mine, lr=lr, eps=opt.param_groups[0]['eps'], betas=opt.param_groups[0]['betas'], fused=True)
    replay = clean_pufferl._DefaultMLPUpdate(pufferlib_b200.namespace(policy=pol2, optimizer=opt2, config=cfg))
    for p, s in zip(mine, st):
        for k in s:
            opt2.state[p][k].copy_(s[k])
    roll = {k: cpu(getattr(exp, k)).copy() for k in ('obs', 'actions', 'logprobs', 'values', 'rewards', 'dones')}
    clean_pufferl.train(data)
    assert data.train_minibatch_path == 'slabs' and data.manual_update.used_fused is False

    ora = oexp.Experience(n * h, bptt, n * h // nm, (16, 16), np.uint8)
    for k, v in roll.items():
        getattr(ora, k)[:] = v
    ora.sort_keys = [(e, t) for t in range(h) for e in range(n)]
    idx = ora.sort_training_data()
    ora.flatten_batch(ogae.compute_gae_f64(ora.dones[idx], ora.values[idx], ora.rewards[idx], cfg.gamma, cfg.gae_lambda))
    m = n * h // nm
    t = lambda a, dtype=torch.float32: torch.as_tensor(np.ascontiguousarray(a).reshape(-1), device=dev).to(dtype)
    replay.pack_heads()
    norms = []
    for epoch in range(cfg.update_epochs):
        for mb in range(nm):
            a64 = ora.b_advantages[mb].astype(np.float64)
            a64 = (a64 - a64.mean()) / (a64.std(ddof=1) + 1e-8)
            batch = pufferlib_b200.namespace(
                obs=torch.as_tensor(ora.b_obs[mb].reshape(m, 16, 16), device=dev), slab_form=False,
                actions=t(ora.b_actions[mb], torch.int64), logprobs=t(ora.b_logprobs[mb]), values=t(ora.b_values[mb]),
                advantages=t(a64), returns=t(ora.b_returns[mb]), row_slab_stride=None, adv_norm=None)
            replay.forward_backward(epoch * nm + mb, cfg.update_epochs * nm, batch, cfg)
            norms.append(float(replay.gflat.double().norm()))
            replay.optimizer_step(cfg)
    torch.cuda.synchronize()
    n_steps = cfg.update_epochs * nm
    assert min(norms) > cfg.max_grad_norm, norms          # every step clipped
    errs = {}
    for k, (p, q) in enumerate(zip(params, mine)):
        errs[f'param{k}'] = float((p.detach() - q.detach()).abs().max())
        for name in ('exp_avg', 'exp_avg_sq'):
            errs[f'{name}{k}'] = rel(opt.state[p][name], opt2.state[q][name])
        assert float(opt.state[p]['step']) == float(opt2.state[q]['step']) == float(n_steps * 2)
    print('replay errors', {k: f'{v:.2e}' for k, v in errs.items()}, flush=True)
    for k in range(6):
        assert errs[f'param{k}'] <= 1e-3 * lr * n_steps, errs
        assert errs[f'exp_avg{k}'] <= 1e-4 and errs[f'exp_avg_sq{k}'] <= 1e-4, errs
    mu = data.manual_update
    w_ref, b_ref = torch.full_like(mu.w_cat, 9.0), torch.full_like(mu.b_cat, 9.0)
    pack_heads([p.detach() for p in params], w_ref, b_ref)
    torch.cuda.synchronize()
    assert torch.equal(mu.w_cat, w_ref) and torch.equal(mu.b_cat, b_ref)
    tot = cpu(replay.loss_means(nm)).astype(np.float64)
    got = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy, data.losses.old_approx_kl,
                    data.losses.approx_kl, data.losses.clipfrac])
    print('losses', got, 'replay', tot, flush=True)
    # the policy loss is a mean of O(1) terms that nearly cancel (normalised advantages have mean 0)
    assert abs(got[0] - tot[0]) <= 1e-6, (got, tot)
    assert np.allclose(got[1:], tot[1:], rtol=1e-4, atol=0), (got, tot)
    clean_pufferl.close(data)

    # pb_adv_norm at C3's size: arrival-order advantages of 65 536 envs x 256 steps, laid out slab-major per minibatch as
    # Experience.flatten_batch_slabs does, normalised per minibatch.  Mean 5: a part of a minibatch left out of the sums
    # moves the mean by ~1e-4 of the std
    n3, h3 = 65536, 256
    g_, r_ = clean_pufferl.slab_layout(n3, h3, nm, bptt)
    m3 = g_ * r_
    gen = torch.Generator(device=dev).manual_seed(5)
    a_tm = torch.randn(n3 * h3, device=dev, generator=gen) + 5.0
    src = a_tm.view(g_, nm, r_).transpose(0, 1).contiguous().view(nm, m3)
    out = torch.full_like(src, float('nan'))
    lib = _native.lib()
    ws = torch.zeros(max(16, lib.pb_adv_norm_workspace_bytes(nm, m3)), dtype=torch.uint8, device=dev)
    _native.check(lib.pb_adv_norm(_native.ptr(src), _native.ptr(out), nm, m3, _native.ptr(ws), ws.numel(),
                                  _native.stream_ptr()))
    rows = torch.as_tensor(clean_pufferl.slab_row_index(n3, h3, nm, bptt), device=dev)
    err = 0.0
    for mb in range(nm):
        a64 = a_tm[rows[mb]].double()
        ref = (a64 - a64.mean()) / (a64.std() + 1e-8)
        err = max(err, float((out[mb].double() - ref).abs().max()))
    print(f'pb_adv_norm at {nm} x {m3} rows: max abs err {err:.2e}', flush=True)
    assert err <= 2e-6, err


# ---- 3. C4 ----------------------------------------------------------------------------------------------------------------
def test_pong_fused_loss_train_matches_reference_loss(monkeypatch):
    """train() on pong (256 envs x 32 steps, bptt 8, 2 minibatches, 2 epochs) with the fused loss (engine 'model': the
    CNN's forward, pb_ppo_loss, autograd) against fused_loss=False (engine 'reference': the policy's forward and the
    reference loss in torch ops), from the same seed: same rollout; b_obs (pb_minibatch_gather, TMA path: 28 224-byte rows)
    bitwise the oracle's flatten_batch; parameters after the update within 2e-5 and losses within 1e-4 relative, the
    chain-vs-autograd precedent.  Observed over the 1 687 719 parameters: max 4.1e-6, 99.9th percentile 2.6e-7; losses
    6.2e-5 relative (approx_kl, 9.6e-6 absolute)."""
    n, h, bptt, nm = 256, 32, 8, 2
    plans = []
    update_plan = clean_pufferl.update_plan
    monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(update_plan(d)) or plans[-1])
    res = {}
    for fused in (True, False):
        vec = pvec.make(ocean.env_creator('pong'), num_envs=n, backend=pvec.B200)
        torch.manual_seed(0)
        pol = cleanrl.Policy(models.Convolutional(vec.driver_env), fused_sample=True, seed=3).cuda()
        data = clean_pufferl.create(ppo_config('pong', n, h, bptt, nm, fused_loss=fused), vec, pol)
        clean_pufferl.evaluate(data)
        exp = data.experience
        roll = {k: cpu(getattr(exp, k)).copy() for k in ('obs', 'actions', 'logprobs', 'values', 'rewards', 'dones')}
        clean_pufferl.train(data)
        plan = plans[-1]
        assert (plan.engine, plan.form, plan.manual) == ('model' if fused else 'reference', 'gathered', None), plan
        ora = oexp.Experience(n * h, bptt, n * h // nm, (4, 84, 84), np.uint8)
        ora.obs[:] = roll['obs']
        ora.sort_keys = [(e, t) for t in range(h) for e in range(n)]
        ora.sort_training_data()
        ora.flatten_batch(np.zeros(n * h, np.float32))
        assert np.array_equal(cpu(exp.b_obs), ora.b_obs)
        losses = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy, data.losses.approx_kl,
                           data.losses.clipfrac, data.losses.explained_variance])
        res[fused] = (roll, [p.detach().clone() for p in pol.parameters()], losses)
        clean_pufferl.close(data)
    for k in res[True][0]:
        assert np.array_equal(res[True][0][k], res[False][0][k]), k
    d = torch.cat([(a - b).abs().flatten() for a, b in zip(res[True][1], res[False][1])]).double()
    q = torch.quantile(d, torch.tensor([0.5, 0.99, 0.999], dtype=torch.float64, device=d.device))
    print(f'parameters ({d.numel()}): max {float(d.max()):.2e} mean {float(d.mean()):.2e} '
          f'quantiles 0.5/0.99/0.999 {[f"{float(v):.2e}" for v in q]}, {int((d > 2e-5).sum())} above 2e-5', flush=True)
    lt, lf = res[True][2], res[False][2]
    print('losses fused', lt, 'reference', lf, flush=True)
    assert float(d.max()) <= 2e-5
    assert np.allclose(lt, lf, rtol=1e-4, atol=1e-6), (lt, lf)


# (row bytes, envs, steps, minibatches, bptt): 28 224 = one (4, 84, 84) pong row, one chunk; 112 896 = fp32 frames, 4
# chunks of 28 224; 30 016 = 2 chunks of 15 008
GATHER = [(28224, 64, 32, 4, 8), (112896, 8, 32, 4, 8), (30016, 24, 16, 4, 4)]


@pytest.mark.parametrize('row_bytes,n,h,nm,bptt', GATHER, ids=[str(g[0]) for g in GATHER])
@pytest.mark.parametrize('sub', ['all', 'middle', 'last'])
def test_minibatch_gather_tma_vs_numpy(row_bytes, n, h, nm, bptt, sub):
    """pb_minibatch_gather on its TMA path (rows >= 4 KiB, 16-byte aligned) against a numpy gather of the oracle's
    b_idxs_obs, for all minibatches and for sub-ranges (mb_begin > 0, mb_count < n_mb); destination rows past the written
    ones hold a canary that must stay untouched."""
    dev = torch.device('cuda')
    mb_begin, mb_count = {'all': (0, nm), 'middle': (1, 2), 'last': (nm - 1, 1)}[sub]
    rows = n * h // (nm * bptt)
    gen = torch.Generator(device=dev).manual_seed(row_bytes + n)
    obs = torch.randint(0, 256, (n * h, row_bytes), dtype=torch.uint8, device=dev, generator=gen)
    n_out, extra = mb_count * rows * bptt, 5
    dst = torch.full((n_out + extra, row_bytes), 0xA5, dtype=torch.uint8, device=dev)
    _native.check(_native.lib().pb_minibatch_gather(_native.ptr(obs), _native.ptr(dst), row_bytes, n, h, nm, rows, bptt,
                                                    mb_begin, mb_count, _native.stream_ptr()))
    torch.cuda.synchronize()
    ora = oexp.Experience(n * h, bptt, n * h // nm, (1,), np.uint8)
    ora.sort_keys = [(e, t) for t in range(h) for e in range(n)]
    ora.sort_training_data()
    want = cpu(obs)[ora.b_idxs_obs[mb_begin:mb_begin + mb_count].reshape(-1)]
    got = cpu(dst)
    bad = int((got[:n_out] != want).any(1).sum())
    print(f'row_bytes={row_bytes} rows={n * h} mb {mb_begin}..{mb_begin + mb_count - 1}: {bad} of {n_out} rows differ',
          flush=True)
    assert bad == 0
    assert (got[n_out:] == 0xA5).all(), 'canary rows written'
