"""Helpers shared by the -m gpu parity tests: thin callers of the C ABI with torch tensors as device memory."""
import ctypes as C

import numpy as np
import torch

from pufferlib_b200 import _native


def mix32(x):
    """pb_mix32 (csrc/pb_common.cuh) on a uint64 array."""
    with np.errstate(over='ignore'):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return (x >> np.uint64(32)).astype(np.uint32)


def uniforms(seed, offset, n):
    """pb_policy_uniform (csrc/policy_sample.cuh) for rows 0..n-1: the uniforms every sampler draws with."""
    with np.errstate(over='ignore'):
        key = (np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(offset) * np.uint64(0xD1B54A32D192ED03)
               + np.arange(n, dtype=np.uint64) * np.uint64(0x2545F4914F6CDD1D))
    return (mix32(key) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def rna(t):
    """Nearest TF32 value (ties away from zero, cvt.rna) of the fp32 value of t, as fp64."""
    bits = t.detach().float().contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32).double()


def trunc_tf32(t):
    """The TF32 value a tensor core reads from the fp32 value of t (low 13 mantissa bits dropped), as fp64."""
    bits = t.detach().float().contiguous().view(torch.int32)
    return (bits & ~0x1FFF).view(torch.float32).double()


# Rounding model of the fp32 accumulation in k_breakout_rollout's tensor-core products (wgmma for the encoder, mma.sync for
# the heads).  The TF32 operand products are exact in fp32 (11 x 11 significant bits), so every error comes from the K = 128
# additions of the products plus the one fp32 add of the bias: each addition loses at most one fp32 ulp of a partial sum
# (2^-23 of it: the adder may truncate rather than round), times 2 because the tensor core aligns a group of addends to the
# largest exponent before it sums them.  Every partial sum is bounded by S = sum_k |x_k w_k| + |b|, so
#     |out_kernel - out_fp64| <= ACC_F32 * S,   ACC_F32 = 2 * (K + 1) * 2^-23.
# This is a worst-case bound: typical errors are about sqrt(K) * 2^-24 * S, some twenty times smaller.
ACC_F32 = 2 * 129 * 2.0 ** -23


def rollout_encoder_ref(x, model):
    """fp64 pre-activation of k_breakout_rollout's encoder for observations x [M, 128]: obs . trunc_tf32(W_enc)^T + b_enc
    (the observations are exact in TF32) -> (pre, bound) with |pre_kernel - pre| <= bound elementwise."""
    w = trunc_tf32(model.encoder.weight)
    b = model.encoder.bias.detach().double()
    x = x.double()
    return x @ w.t() + b, ACC_F32 * (x.abs() @ w.abs().t() + b.abs())


def rollout_heads_ref(hidden, w_cat, b_cat):
    """fp64 head outputs [M, 8] of k_breakout_rollout from fp32 relu(h) [M, 128]: the mma.sync reads relu(h) truncated to
    TF32 and W_heads rounded to TF32 (cvt.rna), and the bias is added in fp32 -> (out, bound), as rollout_encoder_ref."""
    h, w, b = trunc_tf32(hidden), rna(w_cat), b_cat.detach().double()
    return h @ w.t() + b, ACC_F32 * (h.abs() @ w.abs().t() + b.abs())


def check_rollout_dump(dbg_hidden, dbg_out, x0, model, exact_encoder=False):
    """The step-0 dump of k_breakout_rollout (pb_rollout_debug_buffers) checked stage by stage, each stage from the
    kernel's own previous one: relu(h) against the fp64 encoder on the stored step-0 observations x0, then the head
    outputs against fp64 heads recomputed from the dumped relu(h).  Both within the ACC_F32 bound; the padding rows of the
    8-row head matrix are zero, so their outputs must be exactly 0.  exact_encoder: every partial sum of the encoder product
    is exact in fp32 (weights on a coarse grid), so relu(h) must equal fl(sum + b_enc) bit for bit.
    -> (max |err| relu(h), largest bound, max |err| heads, largest bound)."""
    with torch.no_grad():
        pre, bound_h = rollout_encoder_ref(x0, model)
        ref_h = torch.relu(pre)
        err_h = (dbg_hidden.double() - ref_h).abs()
        assert bool((err_h <= bound_h).all()), \
            f'relu(h) at step 0: max err {float(err_h.max()):.3e}, {int((err_h > bound_h).sum())} elements past the bound'
        if exact_encoder:
            off = int((dbg_hidden != ref_h.float()).sum())
            assert off == 0, f'relu(h) at step 0: {off} elements differ from fl(exact sum + b_enc)'
        w_cat, b_cat = model.head_matrix()
        out, bound_o = rollout_heads_ref(dbg_hidden, w_cat, b_cat)
        err_o = (dbg_out.double() - out).abs()
        assert bool((err_o <= bound_o).all()), \
            f'head outputs at step 0: max err per column {[f"{float(v):.2e}" for v in err_o.max(0).values]}, ' \
            f'bound {[f"{float(v):.2e}" for v in bound_o.max(0).values]}'
    return float(err_h.max()), float(bound_h.max()), float(err_o.max()), float(bound_o.max())


def restated_draw(probs, u, window):
    """The inverse-CDF draw of pb_sample_row restated on fp64 probabilities [n, A] (numpy) and the uniforms u [n]:
    -> (actions: the first k with u < cdf_k, near: rows whose u lies within `window` of an inner boundary cdf_k,
    k < A - 1, where the kernel's fp32 weights may decide either way)."""
    cdf = np.cumsum(probs, -1)
    u = np.asarray(u, np.float64)[:, None]
    want = (u >= cdf).sum(-1).clip(max=probs.shape[1] - 1)
    near = (np.abs(u - cdf[:, :-1]) < window).any(-1)
    return want, near


def softmax64(logits):
    """fp64 softmax of logits (a torch tensor, any float type) -> numpy [n, A]."""
    return torch.softmax(logits.double(), -1).cpu().numpy()


def off_boundary_mismatches(actions, logits, seed, offset, window=1e-4):
    """Rows whose action is not the first k with u < cdf_k, among rows with u more than `window` from every cdf_k."""
    want, near = restated_draw(softmax64(logits), uniforms(seed, offset, logits.shape[0]), window)
    return int(((want != np.asarray(actions)) & ~near).sum())


def gae_device(rewards_tm, values_tm, dones_tm, gamma, lam, want_returns=True):
    """rewards/values/dones: numpy [H, N] (arrival order).  Returns (advantages_sorted, returns_sorted) numpy."""
    h, n = rewards_tm.shape
    dev = torch.device('cuda')
    r = torch.as_tensor(np.ascontiguousarray(rewards_tm), device=dev)
    v = torch.as_tensor(np.ascontiguousarray(values_tm), device=dev)
    d = torch.as_tensor(np.ascontiguousarray(dones_tm), device=dev)
    adv = torch.full((n * h,), float('nan'), device=dev)
    ret = torch.full((n * h,), float('nan'), device=dev) if want_returns else None
    lib = _native.lib()
    ws = torch.zeros(max(16, lib.pb_gae_workspace_bytes(n, h)), dtype=torch.uint8, device=dev)
    _native.check(lib.pb_gae(_native.ptr(r), _native.ptr(v), _native.ptr(d), _native.ptr(adv), _native.ptr(ret),
                             n, h, C.c_float(gamma), C.c_float(lam), _native.ptr(ws), ws.numel(),
                             _native.stream_ptr()))
    torch.cuda.synchronize()
    assert int(ws.to(torch.int32).abs().sum()) == 0, 'workspace must be left zeroed'
    return adv.cpu().numpy(), (ret.cpu().numpy() if want_returns else None)


def sorted_from_time_major(x_tm):
    """[H, N] arrival order -> flat sorted order f = e*H + t."""
    return np.ascontiguousarray(x_tm.T).reshape(-1)


def gae_tolerance_check(adv, ref32, ref64):
    """North-star tolerance: fp32 GAE within 1e-5 relative of the reference.  Errors are measured against the float64
    chain on the scale max(1, |A|).  Where the chain is so long and undamped (gamma*lambda ~ 1, no dones) that the
    reference's OWN fp32 rounding exceeds 1e-5, the bar is "no less accurate than 2x the reference's error": two
    fp32 evaluations of an ill-conditioned sum cannot agree better than either is accurate."""
    scale = np.maximum(1.0, np.abs(ref64))
    err = (np.abs(adv.astype(np.float64) - ref64) / scale).max()
    ref_err = (np.abs(ref32.astype(np.float64) - ref64) / scale).max()
    assert err <= max(1e-5, 2 * ref_err), f'cuda err {err:.3e} vs reference fp32 err {ref_err:.3e}'
    direct = (np.abs(adv - ref32) / np.maximum(1.0, np.abs(ref32))).max()
    assert direct <= max(1e-5, err + ref_err), f'direct diff {direct:.3e}'
    return err, ref_err
