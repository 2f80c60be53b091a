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
