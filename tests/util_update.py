"""Checks of the fused wgmma minibatch-update kernel (csrc/mlp_update.cu), shared by tests/test_gpu_update_kernel.py and the
hand-run tests/experimental/check_mlp_update_fused.py.  Not collected by pytest (no test_ prefix).

`case` runs pb_mlp_update_fused on one seeded minibatch and checks it three ways:
  * stage by stage: every stage's reference is computed from the kernel's OWN previous-stage dump (hidden -> dOut -> dPre ->
    gradients), so a mismatch names the stage that is wrong;
  * end to end against an independent float64 autograd restatement of reference clean_pufferl.py:186-244 (the policy of
    models.Default, reference_loss of tests/test_gpu_ppo_loss.py).  Its encoder product takes x and W_enc truncated to TF32,
    as the tensor core does (see reference_update), so it is not an fp32-exact reference and cannot see a wrong TF32
    rounding of the forward operands: only the stage-1 check covers that;
  * the per-block sums of squares the reduce step leaves in the workspace for pb_clip_adam_parts, after every launch.
It covers the arguments the zero-copy train() path passes (Experience.minibatch 'direct'): arrival-order per-row arrays with
row_slab_stride = nm * R and the pointer offset by mb * R (every element of the other minibatches is NaN, so a misindexed read
poisons the gradient), returns formed in the kernel (returns=None), the advantage normalisation applied in the kernel
(adv_norm), and clip_vloss / coefficients other than the benchmark's.
"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pufferlib_b200 import _native  # noqa: E402
from pufferlib_b200.exceptions import APIUsageError  # noqa: E402

CFG = (0.1, 1, 0.1, 0.5, 0.01)       # clip, clip_vloss, vclip, vf_coef, ent_coef (the benchmark's)
CFG_ALT = (0.2, 0, 0.2, 1.0, 0.0)
NDW, TAIL = 128 * 128, 8 * 128 + 128 + 8
X_GAP = 1.0e4                        # x rows that are not in the minibatch: large but finite (see `case`)


def lib():
    return _native.lib()


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def trunc_tf32(t):
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def rna_tf32(t):
    return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def workspace(dev):
    """A workspace for pb_mlp_update_fused with every byte 0xFF: partials the kernel does not write read as NaN."""
    return torch.full((lib().pb_mlp_update_workspace_bytes(),), 0xFF, dtype=torch.uint8, device=dev)


def fused(xbuf, ldx, slab_rows, slab_stride, n_slabs, w_enc, b_enc, w_cat, b_cat, act, olp, adv, ret, oval, n_act, debug,
          dpre_out=None, adv_norm=None, row_stride=None, cfg=CFG, ws=None, gflat=None):
    """One pb_mlp_update_fused launch -> (gflat, stats, hidden, dPre, dOut, workspace); the dumps are None without debug.
    gflat: the gradient buffer to write (else a fresh NaN one); dpre_out: passed through (the library refuses non-null)."""
    dev = xbuf.device
    m = slab_rows * n_slabs
    if gflat is None:
        gflat = torch.full((NDW + TAIL,), float('nan'), device=dev)
    stats = torch.zeros(8, dtype=torch.float64, device=dev)
    if ws is None:
        ws = workspace(dev)
    dh = dp = do = None
    if debug:
        dh = torch.full((m, 128), float('nan'), device=dev)
        dp = torch.full((m, 128), float('nan'), device=dev)
        do = torch.full((m, 8), float('nan'), device=dev)
    _native.check(lib().pb_mlp_update_fused(
        ptr(xbuf), ldx, slab_rows, slab_stride, n_slabs, ptr(w_enc), ptr(b_enc), ptr(w_cat), ptr(b_cat), ptr(act), ptr(olp),
        ptr(adv), ptr(ret), ptr(oval), ptr(adv_norm), slab_rows if row_stride is None else row_stride, n_act, cfg[0], cfg[1],
        cfg[2], cfg[3], cfg[4], ptr(gflat), ptr(stats), ptr(ws), ws.numel(), ptr(dpre_out), ptr(dh), ptr(dp), ptr(do),
        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return gflat, stats, dh, dp, do, ws


def ppo_loss(out, act, olp, adv, ret, oval, n_act, cfg=CFG):
    s = _native.stream_ptr()
    m = out.shape[0]
    dout = torch.empty_like(out)
    stats = torch.empty(8, dtype=torch.float64, device=out.device)
    o, d = out.data_ptr(), dout.data_ptr()
    _native.check(lib().pb_ppo_loss(C.c_void_p(o), 8, C.c_void_p(o + 4 * n_act), 8, ptr(act), ptr(olp), ptr(adv), ptr(ret),
                                    ptr(oval), m, n_act, C.c_float(cfg[0]), cfg[1], C.c_float(cfg[2]), C.c_float(cfg[3]),
                                    C.c_float(cfg[4]), C.c_void_p(d), 8, C.c_void_p(d + 4 * n_act), 8, ptr(stats), s))
    return dout, stats


def rel(a, b):
    return float((a.double() - b.double()).abs().max()) / (float(b.double().abs().max()) + 1e-30)


def check(name, a, b, tol):
    e = rel(a, b)
    print(f'    {name:38s} max err / max|ref| = {e:.3e}  {"ok" if e <= tol else "MISMATCH"}', flush=True)
    return e <= tol


def claim(name, ok):
    print(f'    {name:38s} {"ok" if ok else "MISMATCH"}', flush=True)
    return bool(ok)


def grad_views(gflat, n_act):
    """The six parameter-gradient views _DefaultMLPUpdate hands to the optimizer: W_enc, b_enc, W_dec, b_dec, w_val, b_val."""
    tail = gflat[NDW:]
    dw_cat, db_enc, db_cat = tail[:1024].view(8, 128), tail[1024:1152], tail[1152:]
    return [gflat[:NDW].view(128, 128), db_enc, dw_cat[:n_act], db_cat[:n_act], dw_cat[n_act:n_act + 1],
            db_cat[n_act:n_act + 1]]


def check_sumsq(ws, gflat, n_act):
    """The reduce step's per-block sums of squares (pb_mlp_update_sumsq_offset / _parts): block b holds the fp64 sum of squares
    of partial elements 64b .. 64b + 63, where partial element e < 128 * 128 is dW_enc^T, i.e. gflat[(e % 128) * 128 + e // 128],
    and the rest is the tail of gflat; their total is the squared norm of the six parameter gradients (no padding)."""
    off, n = lib().pb_mlp_update_sumsq_offset(), lib().pb_mlp_update_sumsq_parts()
    sq = ws[off:off + 8 * n].view(torch.float64)
    g = gflat.double()
    elems = torch.cat([g[:NDW].view(128, 128).t().reshape(-1), g[NDW:]])
    elems = torch.cat([elems, elems.new_zeros(64 * n - elems.numel())]).view(n, 64)
    ok = check('sum-of-squares blocks', sq, (elems * elems).sum(1), 1e-12)
    total = sum(float((v.double() ** 2).sum()) for v in grad_views(gflat, n_act))
    ok &= claim(f'sum of squares = |six gradients|^2 ({total:.4e})', abs(float(sq.sum()) - total) <= 1e-12 * total)
    return ok


def reference_update(x, w_enc, b_enc, w_cat, b_cat, n_act, act, olp, adv, ret, oval, cfg):
    """clean_pufferl.py:186-244 for models.Default in float64 autograd -> (gradients of the six parameters, statistics).
    The encoder product takes the operands the tensor core sees (fp32 truncated to TF32, as torch 'high' precision does):
    with fp32 operands the ReLU mask of the ~1e-3 of hidden units that lie within TF32 noise of zero would differ, and each
    such unit moves a whole x * dPre term of dW_enc."""
    import pufferlib_b200
    from test_gpu_ppo_loss import reference_loss
    ns = pufferlib_b200.namespace(clip_coef=cfg[0], clip_vloss=bool(cfg[1]), vf_clip_coef=cfg[2], vf_coef=cfg[3],
                                  ent_coef=cfg[4])
    leaves = [t.double().clone().requires_grad_(True) for t in
              (trunc_tf32(w_enc), b_enc, w_cat[:n_act], b_cat[:n_act], w_cat[n_act:n_act + 1], b_cat[n_act:n_act + 1])]
    we, be, wd, bd, wv, bv = leaves
    with torch.enable_grad():
        hidden = torch.relu(trunc_tf32(x).double() @ we.t() + be)
        loss, st = reference_loss(hidden @ wd.t() + bd, hidden @ wv.t() + bv, act, olp.double(), adv.double(), ret.double(),
                                  oval.double() if oval is not None else None, ns)
        loss.backward()
    return [t.grad for t in leaves], st


def clip_offsets(n, dev):
    """u with |u| in [0, 0.9) on half the rows and in (1.1, 3] on the other half, random sign, float64: a ratio 1 + c u (or a
    value change c u) is inside the clip range [-c, c] on half the rows, outside it on the rest, and never within 0.1 c of
    its edges, far more than the kernel's TF32 noise (~1e-3 on a logit)."""
    inside = torch.rand(n, device=dev) < 0.5
    u = torch.where(inside, 0.9 * torch.rand(n, device=dev), 1.1 + 1.9 * torch.rand(n, device=dev))
    return (u * torch.where(torch.rand(n, device=dev) < 0.5, -1.0, 1.0)).double()


def case(slab_rows, n_slabs, slab_stride, n_act, seed, nm=None, returns=True, old_values=True, adv_norm=False, cfg=CFG,
         ws=None, mb=None, x_tail=64, logit_offset=0.0):
    """One minibatch of `n_slabs` slabs of `slab_rows` rows whose x rows start `slab_stride` rows apart.

    nm (arrival-order rows, as Experience.minibatch 'direct'): the per-row arrays live in buffers of exactly n_slabs * nm
    slabs, the minibatch's slab s at slab s * nm + mb (mb: which of the nm minibatches, default 1), and the kernel gets the
    pointer offset by mb slabs and row_slab_stride = nm * R; every other element is NaN.  Otherwise they are contiguous,
    slab-major.  x_tail: rows of X_GAP after the minibatch's last x slab (0 with mb = nm - 1: the x rows and the per-row
    arrays end flush with their allocations, as the last minibatch of train()'s rollout does).  returns=False: the kernel
    forms raw advantages + old values; old_values=False (needs returns and clip_vloss = 0): no old values at all; adv_norm:
    the kernel normalises the advantages with device constants (mean, 1 / (std + 1e-8)).  ws: a workspace to reuse (else a
    fresh NaN one).  logit_offset: a constant C added to the logit rows of b_cat (C = 1e3: every logit near C, where the
    log-sum-exp lies on the grid of ulp(C) and the unnormalised probabilities miss a sum of 1 by up to ulp(C)/2)."""
    assert (returns or old_values) and (old_values or not cfg[1])
    dev = torch.device('cuda')
    torch.manual_seed(seed)
    m = slab_rows * n_slabs
    if mb is None:
        mb = 1 if nm else 0                                       # the minibatch under test (arrival-order layout)
    assert (0 <= mb < nm) if nm else mb == 0
    if nm:
        assert slab_stride == nm * slab_rows
    total_rows = (n_slabs - 1) * slab_stride + slab_rows
    # x rows outside the minibatch are large and finite: the last tile of a ragged slab loads rows past the slab end into
    # masked rows (0 * x there must stay 0), and a misindexed slab would show up in every gradient
    xbuf = torch.full((mb * slab_rows + total_rows + x_tail, 128), X_GAP, device=dev)
    x = torch.randn(m, 128, device=dev)                           # slab-major rows
    for s in range(n_slabs):
        xbuf[mb * slab_rows + s * slab_stride:][:slab_rows] = x[s * slab_rows:(s + 1) * slab_rows]
    xv = xbuf[mb * slab_rows:]
    w_enc = torch.randn(128, 128, device=dev) * 0.1
    b_enc = torch.randn(128, device=dev) * 0.1
    w_cat = torch.zeros(8, 128, device=dev)
    w_cat[:n_act + 1] = torch.randn(n_act + 1, 128, device=dev) * 0.1
    b_cat = torch.zeros(8, device=dev)
    b_cat[:n_act + 1] = torch.randn(n_act + 1, device=dev) * 0.1
    b_cat[:n_act] += logit_offset
    act = torch.randint(0, n_act, (m,), device=dev)
    # old log-probabilities and old values relative to the float64 policy: rows below, inside and above both clip ranges
    with torch.no_grad():
        h64 = torch.relu(x.double() @ w_enc.double().t() + b_enc.double())
        out64 = h64 @ w_cat.double().t() + b_cat.double()
        nl64 = torch.log_softmax(out64[:, :n_act], 1).gather(1, act[:, None])[:, 0]
    olp = (nl64 - torch.log1p(cfg[0] * clip_offsets(m, dev))).float()
    oval = (out64[:, n_act] + cfg[2] * clip_offsets(m, dev)).float()
    adv = torch.randn(m, device=dev) * 2 + 0.5 if adv_norm else torch.randn(m, device=dev)
    ret = torch.randn(m, device=dev)
    # the returns (or the raw advantages they are formed from) one unit above their draw: the value-head bias gradient is
    # the mean of the residual v - ret, and with a mean near 0 its end-to-end check would measure the cancellation of the
    # rows' TF32 noise rather than the kernel
    if returns:
        ret += 1.0
    else:
        adv += 1.0
    # and returns at least 0.05 from the point where the clipped and unclipped value losses are equal (the midpoint of the
    # new and the clipped value), where the value gradient jumps: shift the returns, or the raw advantages they are formed from
    v64 = out64[:, n_act]
    mid = (v64 + oval.double() + torch.clamp(v64 - oval.double(), -cfg[2], cfg[2])) / 2
    gap = (ret if returns else adv + oval).double() - mid
    shift = torch.where(gap.abs() < 0.05, torch.where(gap < 0, -0.05, 0.05) - gap, torch.zeros_like(gap)).float()
    if returns:
        ret += shift
    else:
        adv += shift
    an = None
    if adv_norm:                      # the constants of Experience.prepare_direct_slabs (pb_adv_stats_slabs)
        a64 = adv.double()
        an = torch.stack([a64.mean(), 1.0 / (a64.std() + 1e-8)]).float()
        a_used = (adv - an[0]) * an[1]                            # the kernel's own fp32 operations: the same bits
    else:
        a_used = adv
    r_used = ret if returns else adv + oval                       # raw advantages + old values (clean_pufferl.py:476-481)
    oval_arg = oval if old_values else None
    # per-row arrays as the kernel reads them
    if nm:
        def rows(t, fill):
            buf = torch.full((n_slabs * nm * slab_rows,), fill, dtype=t.dtype, device=dev)
            buf.view(n_slabs, nm, slab_rows)[:, mb] = t.view(n_slabs, slab_rows)
            return buf[mb * slab_rows:]
        k_act, k_olp, k_adv = rows(act, -1), rows(olp, float('nan')), rows(adv, float('nan'))
        k_ret = rows(ret, float('nan')) if returns else None
        k_oval = rows(oval, float('nan')) if old_values else None
        row_stride = nm * slab_rows
    else:
        k_act, k_olp, k_adv, k_ret, k_oval, row_stride = act, olp, adv, ret if returns else None, oval_arg, slab_rows
    if ws is None:
        ws = workspace(dev)
    print(f'case slab_rows={slab_rows} n_slabs={n_slabs} stride={slab_stride} n_act={n_act} (M={m}) '
          f'nm={nm} mb={mb} x_tail={x_tail} logit_offset={logit_offset} returns={returns} old_values={old_values} '
          f'adv_norm={adv_norm} cfg={cfg}', flush=True)

    def launch(debug, dpre_out=None, gflat=None):
        return fused(xv, 128, slab_rows, slab_stride, n_slabs, w_enc, b_enc, w_cat, b_cat, k_act, k_olp, k_adv, k_ret, k_oval,
                     n_act, debug, dpre_out=dpre_out, adv_norm=an, row_stride=row_stride, cfg=cfg, ws=ws, gflat=gflat)[:5]

    gflat, stats, dh, dp, do = launch(True)
    torch.cuda.synchronize()
    ok = check_sumsq(ws, gflat, n_act)
    # stage 1: forward wgmma (TF32 = truncated operands, fp32 accumulate) + bias + ReLU
    h_ref = torch.relu(trunc_tf32(x).double() @ trunc_tf32(w_enc).double().t() + b_enc.double())
    ok &= check('hidden (forward wgmma)', dh, h_ref, 2e-5)
    # stage 2: heads + loss from the kernel's own hidden; the heads product takes TF32-truncated operands (mma.sync), fp32
    # accumulation
    out = (trunc_tf32(dh).double() @ rna_tf32(w_cat).double().t() + b_cat.double()).float()
    dout_ref, stats_ref = ppo_loss(out, act, olp, a_used, r_used, oval_arg, n_act, cfg)
    ok &= check('dOut (heads + PPO loss)', do, dout_ref, 2e-4)
    ok &= check('loss statistics', stats[:6], stats_ref[:6], 2e-3)
    # stage 3: dPre from the kernel's own dOut and hidden
    dpre_ref = (trunc_tf32(do).double() @ rna_tf32(w_cat).double()) * (dh > 0)
    ok &= check('dPre', dp, dpre_ref, 1e-5)
    # stage 4: gradients from the kernel's own dPre / dOut / hidden
    dw_enc = gflat[:NDW].view(128, 128)
    tail = gflat[NDW:]
    dw_heads, db_enc, db_heads = tail[:1024].view(8, 128), tail[1024:1152], tail[1152:]
    ok &= check('dW_enc (wgmma)', dw_enc, rna_tf32(dp).double().t() @ rna_tf32(x).double(), 2e-5)   # operands rounded to nearest
    ok &= check('dW_heads (mma.sync)', dw_heads, trunc_tf32(do).double().t() @ trunc_tf32(dh).double(), 2e-5)
    ok &= check('db_enc', db_enc, dp.double().sum(0), 2e-5)
    ok &= check('db_heads', db_heads, do.double().sum(0), 2e-5)
    # end to end against float64 autograd: what remains is the epilogue's rounding (TF32 head / dW operands, relative 2^-11
    # per product) -- the TF32 tolerance of the stage checks above; the inputs keep every row away from the edges where a
    # branch of the loss changes, so no row takes another branch than in float64
    grads, st_ref = reference_update(x, w_enc, b_enc, w_cat, b_cat, n_act, act, olp, a_used, r_used, oval_arg, cfg)
    clipfrac = float(st_ref[5])
    ok &= claim(f'rows on both sides of the clip range (clipfrac {clipfrac:.3f})', 0.2 < clipfrac < 0.8)
    views = grad_views(gflat, n_act)
    for name, v, r in zip(('W_enc', 'b_enc', 'W_dec', 'b_dec', 'w_val', 'b_val'), views, grads):
        ok &= check(f'd{name} vs float64 autograd', v, r, 5e-3)
    ok &= claim('padding rows of dW_heads / db_heads exactly 0',
                bool((dw_heads[n_act + 1:] == 0).all()) and bool((db_heads[n_act + 1:] == 0).all()))
    st = stats[:6] / m
    st[1] *= 0.5                       # the kernel sums (v - ret)^2; the loss is half its mean (clean_pufferl.loss_means)
    ok &= check('loss statistics vs float64 autograd', st, st_ref, 2e-3)
    ok &= claim('same clipped rows as float64', round(float(stats[5])) == round(clipfrac * m))
    # a dPre output buffer is refused before any launch: the gradient buffer stays untouched
    g3 = torch.full_like(gflat, float('nan'))
    try:
        launch(False, torch.empty(m, 128, device=dev), g3)
        refused = False
    except APIUsageError:
        refused = True
    torch.cuda.synchronize()
    ok &= claim('non-null dpre_out refused, gradient untouched', refused and bool(torch.isnan(g3).all()))
    # the same launch without the debug dumps must give the same gradients and sums of squares
    g2, s2, _, _, _ = launch(False)
    torch.cuda.synchronize()
    ok &= check('repeat launch (no dumps)', g2, gflat, 1e-6)
    ok &= check_sumsq(ws, g2, n_act)
    return ok


def split_lines(tensors, first):
    """Number of 128-byte lines of `tensors` whose elements k_clip_adam_parts (32 CTAs of 256 threads) updates in more than
    one CTA; `first`: index of the first element of tensors[0] in the concatenated parameters."""
    owners, j = {}, first
    for t in tensors:
        for i in range(t.numel()):
            owners.setdefault((t.data_ptr() + 4 * i) // 128, set()).add((j // 256) % 32)
            j += 1
    return sum(len(o) > 1 for o in owners.values())
