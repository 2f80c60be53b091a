"""pb_clip_adam and pb_clip_adam_parts (csrc/optim.cu) against a float64 restatement of clean_pufferl.py:240-244
(clip_grad_norm_, then torch.optim.Adam(capturable)), one optimizer step at a time from the kernel's own previous fp32 state,
with bounds derived from the kernels' fp32 operations rather than fitted to a run.

Every case is one edge train() can reach: the gradient layouts of _DefaultMLPUpdate.gflat for every hidden size and head-row
count, gradients on both sides of eps, step counters loaded from a checkpoint, the hyper-parameters of the param group, grad
scales 1 / world, the clip boundary, the kernels' size limits, and the multi-CTA kernel's CTA boundaries and step bookkeeping
over back-to-back launches and graph replays."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from pufferlib_b200 import _native
from pufferlib_b200.exceptions import APIUsageError

pytestmark = pytest.mark.gpu

U = 2.0 ** -24            # unit roundoff of fp32 (round to nearest): one fp32 operation is off by at most U relative
KERNELS = ['single_cta', 'parts']
N_PARTS = 257             # partial sums of squares handed to pb_clip_adam_parts (one more than its CTA's 256 threads)


def f32(x):
    """x as the fp32 value the kernel receives (every hyper-parameter crosses the C ABI as a float)."""
    return float(np.float32(x))


def gflat_views(hid, rows, n_act, features):
    """(offset, numel) of the six gradient views of _DefaultMLPUpdate.gflat (dW_enc | dW_cat[rows x hid] | db_enc |
    db_cat[rows]), in parameter order W_enc, b_enc, W_dec, b_dec, w_val, b_val, sliced as _DefaultMLPUpdate.__init__
    slices them; and the buffer's length."""
    gflat = torch.zeros(hid * features + rows * hid + hid + rows)
    dw_enc = gflat[:hid * features].view(hid, features)
    tail = gflat[hid * features:]
    dw_cat = tail[:rows * hid].view(rows, hid)
    db_enc, db_cat = tail[rows * hid:(rows + 1) * hid], tail[(rows + 1) * hid:]
    grads = [dw_enc, db_enc, dw_cat[:n_act], db_cat[:n_act], dw_cat[n_act:n_act + 1], db_cat[n_act:n_act + 1]]
    return [(g.storage_offset(), g.numel()) for g in grads], gflat.numel()


def packed_views(sizes):
    offs = np.cumsum([0] + list(sizes))
    return [(int(o), int(n)) for o, n in zip(offs, sizes)], int(offs[-1])


class Case:
    """One optimizer and the gradients of `steps` consecutive steps.  Parameters are of the size of one Adam step (lr), so
    the parameter check resolves the update to a few fp32 ulps instead of hiding it under the rounding of a much larger
    parameter.  State loaded at step0 > 0 carries moments from three float64 steps on random gradients, as after
    optimizer.load_state_dict(); step0 = 0 is a fresh optimizer (zero moments).

    Gradients are normal with standard deviation `scale`, or (loguniform) of magnitude log-uniform over 1e-9 .. 1e-2 with
    10 % exact zeros at the same elements every step; zero_tensor: one gradient view that is zero throughout.  clip: the
    max_norm of each step as a multiple of that step's float64 norm (0.5 when the norm is 0).  The padding of the flat
    buffer outside the views is NaN: a kernel that reads it poisons the norm and every update."""

    def __init__(self, views, flat_n, seed, *, steps=2, step0=0, scale=0.05, loguniform=False, zero_tensor=None,
                 betas=(0.9, 0.999), eps=1e-5, lr_dev=True, world=1, clip=(2.0, 0.5), head=None):
        rng = np.random.default_rng(seed)
        self.views, self.flat_n, self.head = views, flat_n, head
        self.sizes = [n for _, n in views]
        self.b1, self.b2, self.eps, self.lr_dev = f32(betas[0]), f32(betas[1]), f32(eps), lr_dev
        self.grad_scale = f32(1.0 / world)
        step0 = step0 if isinstance(step0, (list, tuple)) else [step0] * len(views)
        self.step0 = [f32(s) for s in step0]
        self.p = [(rng.standard_normal(n) * 2.5e-4).astype(np.float32) for n in self.sizes]
        self.m, self.v = [], []
        for n, s in zip(self.sizes, step0):
            m, v = np.zeros(n), np.zeros(n)
            for _ in range(3 if s > 0 else 0):
                g = rng.standard_normal(n) * 0.05
                m, v = self.b1 * m + (1 - self.b1) * g, self.b2 * v + (1 - self.b2) * g * g
            self.m.append(m.astype(np.float32))
            self.v.append(v.astype(np.float32))
        zero = [rng.random(n) < 0.1 for n in self.sizes] if loguniform else None
        self.grads, self.max_norm, self.lr = [], [], []
        for k in range(steps):
            flat = np.full(flat_n, np.nan, dtype=np.float32)
            for t, (o, n) in enumerate(views):
                if loguniform:
                    g = np.where(zero[t], 0.0, np.sign(rng.standard_normal(n)) * 10.0 ** rng.uniform(-9, -2, n))
                else:
                    g = rng.standard_normal(n) * scale
                flat[o:o + n] = 0.0 if t == zero_tensor else g
            self.grads.append(flat)
            norm = self.grad_scale * math.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in self.views_of(flat)))
            self.max_norm.append(f32(clip[k % len(clip)] * norm) if norm > 0 else 0.5)
            self.lr.append(f32(2.5e-4 * (1 - k / steps)))      # changed between steps, as anneal_lr does

    def views_of(self, flat):
        return [flat[o:o + n] for o, n in self.views]


# ---- the float64 oracle and the bounds on the kernels' deviation from it

def adam64(p, m, v, step, g, coef, lr, b1, b2, eps, ep=0.0, em=0.0, rv=0.0):
    """One step of torch.optim.Adam(capturable) in float64 after clip_grad_norm_: step += 1 first, then the bias
    corrections, the first moment in lerp form; g the fp32 gradient, coef the clip coefficient times grad_scale.

    Also returns bounds on how far the fp32 kernel, started from a state within (ep, em, rv) of (p, m, v) -- absolute for p
    and m, relative for v -- can land from the float64 result.  Each bound follows the kernel's fp32 operations (each off by
    at most U relative; FMA contraction only removes roundings):
      x  = g * fl(coef * grad_scale)                          2 roundings: |x - x64| <= 2U |x64|
      m' = m + w1 (x - m)      (w1 = 1 - beta1, exact)        x's 2U, the difference, product and sum: to first order
                                                              U (5 w1 |x| + (1 + w1) |m|); 6U (|m| + w1 |x|) leaves one U
                                                              for the second-order terms
      v' = beta2 v + w2 x x                                   all terms >= 0: x^2 4U, two products, one sum -> (1 + U)^7;
                                                              the carried-in v term (1 + rv)(1 + U)^2
      den = sqrt(v') / fl(sqrt(bc2)) + eps                    sqrt(1 +- rv'), then the sqrt, fl(sqrt(bc2)), division and sum
      q  = fl(fl(lr / bc1) * m') / den                        3 roundings and den's: ratio within F = (1 + U)^3 / (1 - ed),
                                                              plus the carried-in m' error at lr / bc1 / den
      p' = fl(p - q)                                          half an fp32 ulp at |p'| + the errors above
    The bias corrections are formed in float64 and differ from the oracle's by < 1e3 float64 ulps, far below U."""
    step = step + 1.0
    w1, w2 = 1.0 - b1, 1.0 - b2
    x = g * coef
    m1 = m + w1 * (x - m)
    v1 = b2 * v + w2 * x * x
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    step_size = lr / bc1
    den = np.sqrt(v1) / math.sqrt(bc2) + eps
    p1 = p - step_size * m1 / den
    em1 = b1 * em + 6 * U * (np.abs(m) + em + w1 * np.abs(x))
    rv1 = np.maximum((1 + rv) * (1 + U) ** 2, (1 + U) ** 7) - 1
    ed = np.maximum(np.sqrt(1 + rv1) * (1 + U) ** 3 / (1 - U) - 1, 1 - np.sqrt(1 - rv1) * (1 - U) ** 3 / (1 + U))
    F = (1 + U) ** 3 / (1 - ed)
    eq = step_size / den * (em1 * F + np.abs(m1) * (F - 1))
    ep1 = ep + eq
    ep1 = ep1 + half_ulp(np.abs(p1) + ep1)
    return (p1, m1, v1, step), (ep1, em1, rv1)


def half_ulp(a):
    """Half the fp32 spacing at magnitude a, taken at a rounded to fp32: no fp32 value of magnitude <= a has a larger one."""
    return np.spacing(np.abs(a).astype(np.float32)).astype(np.float64) / 2


def clip_coef(max_norm, norm):
    """The kernels' clip coefficient from their reported norm, in fp32 as they form it: min(max_norm / (norm + 1e-6), 1).
    The oracle takes it from the kernel's norm, not its own: the two norms can fall on different sides of the clip
    boundary, and the norm check bounds their difference."""
    return min(np.float32(max_norm) / (np.float32(norm) + np.float32(1e-6)), np.float32(1.0))


def norm_bound(kernel, sizes):
    """Relative bound on the reported norm against the float64 norm of the fp32 gradients times grad_scale.
    k_clip_adam: each of 1024 threads sums its J <= K = sum(ceil(numel / 1024)) squares of fl(g * grad_scale) in fp32
    (the scaling, the square and J - 1 additions of terms >= 0: (J + 2) U relative), the threads' sums add in float64,
    the square root halves the relative error and the cast to fp32 adds U: (K + 2) U / 2 + U, and U / 2 for the
    second-order and float64 terms.  k_clip_adam_parts: float64 partial sums, then fp32 rounding of the root and the
    product with grad_scale: 2 U, and U / 2 as above."""
    if kernel == 'single_cta':
        k = sum(-(-n // 1024) for n in sizes)
        return (k / 2 + 2.5) * U
    return 2.5 * U


def assert_within(what, got, ref, bound):
    err = np.abs(got - ref)
    bad = ~(err <= bound)                     # a NaN is outside every bound
    assert not bad.any(), (f'{what}: {int(bad.sum())} of {bad.size} elements outside the bound, worst error / bound '
                           f'{float(np.nanmax(err / np.maximum(bound, 1e-300))):.3g}')


# ---- running the kernels

class Device:
    """A Case on the GPU: every parameter and state tensor its own allocation (as the nn.Linear weights and biases of a
    models.Default are), the gradients views of one flat buffer."""

    def __init__(self, case, kernel, n_parts=N_PARTS):
        dev = torch.device('cuda')
        self.case, self.kernel, self.n_parts = case, kernel, n_parts
        self.p = [torch.tensor(a, device=dev) for a in case.p]
        self.m = [torch.tensor(a, device=dev) for a in case.m]
        self.v = [torch.tensor(a, device=dev) for a in case.v]
        self.step = [torch.tensor(s, dtype=torch.float32, device=dev) for s in case.step0]
        self.flat = torch.full((case.flat_n,), float('nan'), device=dev)
        self.lr_t = torch.zeros((), device=dev)
        self.norm = torch.full((1,), float('nan'), device=dev)
        self.parts = torch.zeros(n_parts, dtype=torch.float64, device=dev)
        self.tensors = self.adam_tensors(self.flat)
        self.pack = None
        if kernel == 'parts' and case.head is not None and case.head[1] <= 7:
            hid, n_act = case.head
            self.w_cat, self.b_cat = torch.full((8, hid), 9.0, device=dev), torch.full((8,), 9.0, device=dev)
            self.pack = _native.HeadPack(*(self.p[k].data_ptr() for k in (2, 3, 4, 5)), self.w_cat.data_ptr(),
                                         self.b_cat.data_ptr(), n_act, hid)

    def adam_tensors(self, flat):
        arr = (_native.AdamTensor * len(self.p))()
        for k, (o, n) in enumerate(self.case.views):
            arr[k] = _native.AdamTensor(self.p[k].data_ptr(), self.m[k].data_ptr(), self.v[k].data_ptr(),
                                        self.step[k].data_ptr(), flat.data_ptr() + 4 * o, n)
        return arr

    def sumsq_parts(self, flat):
        """The unscaled gradient's sum of squares as float64 partial sums over tensor_split chunks of the six views."""
        g = torch.cat([flat[o:o + n] for o, n in self.case.views]).double()
        return torch.stack([(c * c).sum() for c in torch.tensor_split(g, self.n_parts)])

    def launch(self, k, tensors=None, parts=None):
        c, lib = self.case, _native.lib()
        hyper = (C.c_float(c.max_norm[k]), C.c_float(c.grad_scale), C.c_float(0.0 if c.lr_dev else c.lr[k]),
                 _native.ptr(self.lr_t) if c.lr_dev else None, C.c_float(c.b1), C.c_float(c.b2), C.c_float(c.eps),
                 _native.ptr(self.norm))
        tensors = self.tensors if tensors is None else tensors
        if self.kernel == 'single_cta':
            _native.check(lib.pb_clip_adam(tensors, len(self.p), *hyper, _native.stream_ptr()))
        else:
            _native.check(lib.pb_clip_adam_parts(tensors, len(self.p), *hyper, _native.ptr(self.parts if parts is None else parts),
                                                 self.n_parts, None, None if self.pack is None else C.byref(self.pack),
                                                 _native.stream_ptr()))

    def state(self):
        f = lambda ts: [t.cpu().numpy().astype(np.float64) for t in ts]
        return f(self.p), f(self.m), f(self.v), [float(s) for s in self.step]

    def check_pack(self, what):
        if self.pack is None:
            return
        hid, n_act = self.case.head
        w_ref, b_ref = torch.full_like(self.w_cat, 7.0), torch.full_like(self.b_cat, 7.0)
        _native.check(_native.lib().pb_pack_heads(*(_native.ptr(self.p[k]) for k in (2, 3, 4, 5)), n_act, hid,
                                                  _native.ptr(w_ref), _native.ptr(b_ref), None, None, 0, _native.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(self.w_cat, w_ref) and torch.equal(self.b_cat, b_ref), f'{what}: head matrix'


def check_norm(kernel, case, flat, norm_k, what):
    norm64 = case.grad_scale * math.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in case.views_of(flat)))
    assert abs(norm_k - norm64) <= norm_bound(kernel, case.sizes) * norm64, (what, norm_k, norm64)


def run(case, kernel, n_parts=N_PARTS):
    """Each step: copy the kernel's fp32 state, launch, then compare with the oracle's step from that copy."""
    d = Device(case, kernel, n_parts)
    for k, flat in enumerate(case.grads):
        what = f'{kernel} step {k + 1}'
        d.flat.copy_(torch.from_numpy(flat))
        d.lr_t.fill_(case.lr[k])
        d.parts.copy_(d.sumsq_parts(d.flat))
        p0, m0, v0, s0 = d.state()
        d.launch(k)
        torch.cuda.synchronize()
        p1, m1, v1, s1 = d.state()
        norm_k = float(d.norm)
        check_norm(kernel, case, flat, norm_k, what)
        coef = float(clip_coef(case.max_norm[k], norm_k)) * case.grad_scale
        for t, g in enumerate(case.views_of(flat)):
            (pr, mr, vr, sr), (ep, em, rv) = adam64(p0[t], m0[t], v0[t], s0[t], g.astype(np.float64), coef, case.lr[k],
                                                    case.b1, case.b2, case.eps)
            assert s1[t] == f32(sr), (what, t, s1[t], sr)
            assert_within(f'{what} tensor {t} exp_avg', m1[t], mr, em)
            assert_within(f'{what} tensor {t} exp_avg_sq', v1[t], vr, rv * vr)
            assert_within(f'{what} tensor {t} param', p1[t], pr, ep)
            # no gradient and no moments: the moments stay 0 and the parameter keeps its bits
            idle = (g == 0) & (m0[t] == 0) & (v0[t] == 0)
            assert (m1[t][idle] == 0).all() and (v1[t][idle] == 0).all() and (p1[t][idle] == p0[t][idle]).all(), what
        d.check_pack(what)
    return d


# ---- the layouts train() builds: six views of gflat for every hidden size, head-row count and action count

LAYOUTS = [  # hid, rows, n_act, features
    (128, 8, 1, 128), (128, 8, 7, 128), (128, 8, 7, 49), (128, 16, 8, 1), (128, 16, 15, 128), (128, 32, 16, 49),
    (128, 32, 31, 1), (256, 8, 1, 49), (256, 8, 7, 1), (256, 16, 8, 128), (256, 16, 15, 49), (256, 32, 31, 128),
    (384, 8, 1, 1), (384, 8, 7, 128), (384, 16, 15, 1), (384, 32, 16, 128), (512, 8, 7, 49), (512, 16, 8, 49),
    (512, 32, 16, 1), (512, 32, 31, 128)]


def default_case(hid, rows, n_act, features, seed, **kw):
    views, flat_n = gflat_views(hid, rows, n_act, features)
    return Case(views, flat_n, seed, head=(hid, n_act), **kw)


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('hid,rows,n_act,features', LAYOUTS, ids=[f'hid{h}-rows{r}-act{a}-f{f}' for h, r, a, f in LAYOUTS])
def test_gflat_layouts(hid, rows, n_act, features, kernel):
    """Step 1 unclipped, step 2 clipped; the value bias is one element at an odd float offset when n_act is odd."""
    run(default_case(hid, rows, n_act, features, seed=hid + 7 * n_act + features), kernel)


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('eps', [1e-5, 1e-8])
def test_gradients_around_eps(eps, kernel):
    """Gradient magnitudes log-uniform over 1e-9 .. 1e-2 from a fresh optimizer, so the bias-corrected sqrt(v) lies below,
    at and above eps; exact zeros (no moments, no update) and a whole zero tensor (b_enc)."""
    run(default_case(128, 8, 5, 128, seed=11, steps=3, loguniform=True, zero_tensor=1, eps=eps, clip=(10.0,)), kernel)


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('step0', [0, 1, 9, 999, 123456, 2 ** 20])
def test_step_counter_loaded_from_checkpoint(step0, kernel):
    """The bias corrections from 1 - beta^step near 0.1 / 0.001 (step 1) to exactly 1 in float64 (2^20)."""
    run(default_case(128, 8, 4, 128, seed=step0 % 1000, step0=step0), kernel)


HYPER = [((0.9, 0.999), 1e-5, False), ((0.9, 0.999), 1e-8, True), ((0.0, 0.99), 1e-5, True), ((0.0, 0.99), 1e-8, False),
         ((0.5, 0.9), 1e-5, False), ((0.5, 0.9), 1e-8, True)]


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('betas,eps,lr_dev', HYPER,
                         ids=[f'b{b1}-{b2}-eps{e}-lr_{"device" if d else "host"}' for (b1, b2), e, d in HYPER])
def test_param_group_hyper_parameters(betas, eps, lr_dev, kernel):
    """Whatever the param group holds; the learning rate changes between steps, on the host or in a device tensor."""
    run(default_case(256, 8, 3, 49, seed=5, steps=3, step0=9, betas=betas, eps=eps, lr_dev=lr_dev), kernel)


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('world', [1, 2, 3, 8])
def test_grad_scale_one_over_world(world, kernel):
    """grad_scale = fl(1 / world) scales the summed gradient before the norm, also when it is not a power of two."""
    run(default_case(128, 8, 6, 128, seed=world, world=world, scale=0.05 * world), kernel)


CLIP = {'norm_above_max_by_2^-20': dict(clip=(1 / (1 + 2.0 ** -20),)),
        'norm_below_max_by_2^-20': dict(clip=(1 / (1 - 2.0 ** -20),)),
        'norm_1e6_times_max': dict(clip=(1e-6,)),
        'all_zero_gradients': dict(scale=0.0, step0=9)}


@pytest.mark.parametrize('kernel', KERNELS)
@pytest.mark.parametrize('edge', list(CLIP))
def test_clip_boundary(edge, kernel):
    """Gradient norms near 65, so the 1e-6 in the coefficient's denominator is far below 2^-20 of it; with zero gradients
    the norm is exactly 0, the coefficient 1 and only the loaded first moment moves the parameters."""
    run(default_case(128, 8, 3, 128, seed=17, **{'scale': 0.5, **CLIP[edge]}), kernel)


# ---- the limits

@pytest.mark.parametrize('kernel', KERNELS)
def test_one_tensor_of_2_20_elements(kernel):
    """The single-CTA kernel's largest input: 1024 squares per thread in fp32 before the float64 reduce."""
    views, flat_n = packed_views([1 << 20])
    run(Case(views, flat_n, seed=3, steps=1, clip=(0.5,)), kernel)


def test_size_and_tensor_count_refused():
    """2^20 + 1 elements (pb_clip_adam only) and 9 tensors are refused before any launch: the state stays as it was."""
    dev = torch.device('cuda')
    lib = _native.lib()

    def tensors(sizes):
        ts = [torch.zeros(n, device=dev) for n in sizes]
        step = torch.zeros((), device=dev)
        arr = (_native.AdamTensor * len(sizes))()
        for k, t in enumerate(ts):
            arr[k] = _native.AdamTensor(t.data_ptr(), t.data_ptr(), t.data_ptr(), step.data_ptr(), t.data_ptr(), t.numel())
        return arr, ts, step

    hyper = (C.c_float(0.5), C.c_float(1.0), C.c_float(2.5e-4), None, C.c_float(0.9), C.c_float(0.999), C.c_float(1e-5), None)
    parts = torch.ones(1, dtype=torch.float64, device=dev)
    arr, ts, step = tensors([(1 << 20) + 1])
    with pytest.raises(NotImplementedError):
        _native.check(lib.pb_clip_adam(arr, 1, *hyper, _native.stream_ptr()))
    arr9, ts9, step9 = tensors([16] * 9)
    with pytest.raises(APIUsageError):
        _native.check(lib.pb_clip_adam(arr9, 9, *hyper, _native.stream_ptr()))
    with pytest.raises(APIUsageError):
        _native.check(lib.pb_clip_adam_parts(arr9, 9, *hyper, _native.ptr(parts), 1, None, None, _native.stream_ptr()))
    torch.cuda.synchronize()
    assert float(step) == 0.0 and float(step9) == 0.0
    assert all(not t.any() for t in ts + ts9)


# ---- eight tensors (CA_MAX_TENSORS) at odd sizes: the multi-CTA kernel's CTA boundaries inside and between tensors

EIGHT = [1, 3, 255, 256, 257, 8191, 8192, 8193]        # 25 348 elements: not a multiple of 32 CTAs x 256 threads
EIGHT_STEPS = [0, 1, 2, 9, 999, 123456, 2 ** 20, 5]    # one step counter per tensor, each with its own bias corrections


@pytest.mark.parametrize('kernel,n_parts', [('single_cta', N_PARTS)] + [('parts', n) for n in (1, 255, 256, 257, 4096)],
                         ids=['single_cta'] + [f'parts-n_parts{n}' for n in (1, 255, 256, 257, 4096)])
def test_eight_tensors_of_odd_sizes(kernel, n_parts):
    views, flat_n = packed_views(EIGHT)
    run(Case(views, flat_n, seed=n_parts, step0=EIGHT_STEPS), kernel, n_parts)


# ---- the multi-CTA kernel's step bookkeeping (g_cap_ticket) over many launches without a host sync

@pytest.mark.parametrize('mode', ['back_to_back', 'graph_replays'])
def test_parts_fifty_steps_without_host_sync(mode):
    """50 optimizer steps of the fused train() configuration (hidden 128, 5 actions, head pack) on one stream: launched
    back to back, each on its own gradients, or one step captured in a CUDA graph and replayed 50 times with the inputs
    copied in between, as the captured train() graph replays its optimizer step.  Every step counter ends at exactly 50,
    the head matrix is the pack of the final parameters, and the final state is within the bounds of 50 float64 steps
    chained from the initial state, each bound carried through the next step by adam64."""
    steps = 50
    case = default_case(128, 8, 5, 128, seed=50, steps=steps, clip=(1e3,))      # no clipping: coefficient exactly 1
    d = Device(case, 'parts', _native.lib().pb_mlp_update_sumsq_parts())
    dev = d.flat.device
    grads = torch.from_numpy(np.stack(case.grads)).to(dev)
    parts = torch.stack([d.sumsq_parts(g) for g in grads])
    lrs = torch.tensor(case.lr, device=dev)
    torch.cuda.synchronize()
    if mode == 'back_to_back':
        tensors = [d.adam_tensors(g) for g in grads]
        for k in range(steps):
            d.lr_t.copy_(lrs[k])
            d.launch(k, tensors[k], parts[k])
    else:
        case.max_norm = [case.max_norm[0]] * steps        # one captured launch: the same max_norm every replay
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            d.launch(0)
        for k in range(steps):
            d.flat.copy_(grads[k])
            d.parts.copy_(parts[k])
            d.lr_t.copy_(lrs[k])
            graph.replay()
    torch.cuda.synchronize()
    p1, m1, v1, s1 = d.state()
    assert s1 == [50.0] * len(s1)
    check_norm('parts', case, case.grads[-1], float(d.norm), 'last step')
    d.check_pack('after 50 steps')
    for t in range(len(case.sizes)):
        st = (case.p[t].astype(np.float64), case.m[t].astype(np.float64), case.v[t].astype(np.float64), 0.0)
        err = (0.0, 0.0, 0.0)
        for k in range(steps):
            norm64 = case.grad_scale * math.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in case.views_of(case.grads[k])))
            assert case.max_norm[k] >= 1e2 * norm64
            st, err = adam64(*st, case.views_of(case.grads[k])[t].astype(np.float64), case.grad_scale, case.lr[k],
                             case.b1, case.b2, case.eps, *err)
        assert_within(f'tensor {t} exp_avg after 50 steps', m1[t], st[1], err[1])
        assert_within(f'tensor {t} exp_avg_sq after 50 steps', v1[t], st[2], err[2] * st[2])
        assert_within(f'tensor {t} param after 50 steps', p1[t], st[0], err[0])
