"""models.Convolutional's first layer on the uint8 frames (csrc/nature_conv1.cu): pb_conv1_u8_forward and
pb_conv1_u8_wgrad against exact restatements and fp64, their ABI refusals, determinism and capture, the model's fast path
against the stock path, and train() on pong with it (C4 at full size included).

Bounds.  The forward's S = sum_k w_k x_k takes w rounded to TF32 (relative 2^-11) and x exact, in 32 mma k-steps of 8
fp32-accumulated products, then y = relu(fma(S, fl(1/255), b)): |y - y64| <= (2^-11 + 48 * 2^-24) * conv(x, |w|) / 255
+ 2^-23 * |y64| + 2^-23 * |b| (relu is 1-Lipschitz).  The weight gradient takes dz rounded to TF32 (2^-11) and x exact;
each CTA accumulates n_cta = 50 * rows-per-CTA mma steps, scales by fl(1/255), and k_reduce_partials adds ceil(G / 32)
terms per lane and a 5-level tree: |dW - dW64| <= (2^-11 + (n_cta + ceil(G / 32) + 16) * 2^-24) * sum |dz| x / 255;
db sums fp32 dz (16 values per lane and row, then a 5-level shuffle tree, then the reduce)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pufferlib_b200 import _native, models
from pufferlib_b200.exceptions import APIUsageError

pytestmark = pytest.mark.gpu

ROW = 4 * 84 * 84
Y_ROW = 32 * 400
WG_CTAS = 264
INV255 = np.float32(1.0) / np.float32(255.0)
U = 2.0 ** -24


def lib():
    return _native.lib()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def frames(m, stride, seed, poison_rows=2):
    """m rows of (4, 84, 84) uint8, `stride` bytes apart, followed by `poison_rows` rows of 255 that must never be read;
    rows 0 and 1 (when present) all 0 and all 255."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    buf = torch.randint(0, 256, ((m + poison_rows) * stride,), dtype=torch.uint8, device='cuda', generator=gen)
    rows = buf.view(m + poison_rows, stride)
    rows[m:] = 255
    if m > 2:
        rows[0] = 0
        rows[1] = 255
    x = torch.as_strided(buf, (m, 4, 84, 84), (stride, 7056, 84, 1))
    return x


def forward(x, w, b, canary=2):
    m = x.shape[0]
    yb = torch.full(((m + canary) * Y_ROW,), -7.0, device='cuda')
    _native.check(lib().pb_conv1_u8_forward(_native.ptr(x), x.stride(0), m, _native.ptr(w), _native.ptr(b),
                                            _native.ptr(yb), _native.stream_ptr()))
    assert bool((yb[m * Y_ROW:] == -7.0).all()), 'rows after y were written'
    return yb[:m * Y_ROW].view(m, 32, 20, 20)


def wgrad(x, y, dy):
    m = x.shape[0]
    dw = torch.full((32, 256), float('nan'), device='cuda')
    db = torch.full((32,), float('nan'), device='cuda')
    ws = torch.full((lib().pb_conv1_u8_wgrad_workspace_bytes(m),), 0xFF, dtype=torch.uint8, device='cuda')
    _native.check(lib().pb_conv1_u8_wgrad(_native.ptr(x), x.stride(0), m, _native.ptr(y), _native.ptr(dy), _native.ptr(dw),
                                          _native.ptr(db), _native.ptr(ws), ws.numel(), _native.stream_ptr()))
    return dw, db


def cols64(x):
    """x_col [B, 256, 400] in fp64, k = c*64 + ky*8 + kx."""
    return F.unfold(x.double(), 8, stride=4)


def chunks(m, size=2048):
    return [(lo, min(m, lo + size)) for lo in range(0, m, size)]


def reduce_ref(parts):
    """k_reduce_partials restated in fp32: lane l sums partial rows l, l + 32, ... in order, then the xor tree."""
    lanes = np.zeros((32,) + parts.shape[1:], np.float32)
    for b_ in range(parts.shape[0]):
        lanes[b_ % 32] = lanes[b_ % 32] + parts[b_]
    for off in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ off]
    return lanes[0]


def grid_weights(seed):
    rng = np.random.default_rng(seed)
    w = rng.integers(-64, 65, (32, 256)).astype(np.float32) / 256      # 2^-8 grid, |w| <= 0.25
    b = rng.integers(-64, 65, 32).astype(np.float32) / 256
    return torch.as_tensor(w, device='cuda'), torch.as_tensor(b, device='cuda')


def orthogonal_weights(seed):
    torch.manual_seed(seed)
    conv = models.layer_init(torch.nn.Conv2d(4, 32, 8, stride=4)).cuda()
    with torch.no_grad():
        conv.bias.uniform_(-0.5, 0.5)
    return conv.weight.detach().reshape(32, 256).contiguous(), conv.bias.detach().clone()


# ---- 1. exact case ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('m', [1, 3, 37])
def test_exact_forward_and_wgrad_bitwise(m):
    """W, b and dy on the 2^-8 grid (|w| <= 0.25, |dy| <= 0.25): every TF32 operand and every partial sum is exact, so
    y must equal relu(fl32(S * fl32(1/255) + b)) (the fma of the epilogue; S the exact integer-grid sum, the fp64
    expression exact) bit for bit.  With m <= 264 every weight-gradient CTA owns one row: its partial is
    fl32(S_row * fl32(1/255)) of the exact row sum, summed by k_reduce_partials' order (reduce_ref); db = the exact sum."""
    w, b = grid_weights(m)
    x = frames(m, ROW, seed=m)
    y = forward(x, w, b)
    xc = cols64(x)                                                             # [m, 256, 400]
    s = torch.einsum('ck,bkp->bcp', w.double(), xc)                            # exact
    pre = (s * float(INV255) + b.double()[None, :, None]).float()
    want = torch.relu(pre).view(m, 32, 20, 20)
    assert torch.equal(y, want), float((y - want).abs().max())

    rng = np.random.default_rng(100 + m)
    dy = torch.as_tensor(rng.integers(-64, 65, (m, 32, 20, 20)).astype(np.float32) / 256, device='cuda')
    dw, db = wgrad(x, y, dy)
    dz = (dy * (y > 0)).double().view(m, 32, 400)
    s_rows = torch.einsum('bcp,bkp->bck', dz, xc)                              # exact per row
    parts = (s_rows * float(INV255)).float().cpu().numpy().reshape(m, -1)
    want_dw = reduce_ref(parts).reshape(32, 256)
    assert np.array_equal(dw.cpu().numpy(), want_dw)
    assert torch.equal(db, dz.sum((0, 2)).float())


# ---- 2. general case against fp64 -------------------------------------------------------------------------------------
def general_sizes():
    g = 2 * sms()
    return sorted({1, 2, g - 1, g, g + 1, 2 * g + 1, 4096})


def check_general(m, stride, seed):
    w, b = orthogonal_weights(seed)
    x = frames(m, stride, seed)
    y = forward(x, w, b)
    gen = torch.Generator(device='cuda').manual_seed(seed + 1)
    dy = torch.randn(m, 32, 20, 20, device='cuda', generator=gen)
    dyb = torch.full(((m + 2) * Y_ROW,), 1.0e6, device='cuda')                 # canary rows: huge gradients
    dyb[:m * Y_ROW] = dy.reshape(-1)
    yb = torch.full(((m + 2) * Y_ROW,), 1.0, device='cuda')
    yb[:m * Y_ROW] = y.reshape(-1)
    dw, db = wgrad(x, yb[:m * Y_ROW].view(m, 32, 20, 20), dyb[:m * Y_ROW].view(m, 32, 20, 20))
    w64, wt = w.double(), torch.as_tensor(w.cpu().numpy(), device='cuda').double().abs()
    fwd_frac, dw64, dwabs, db64, dbabs = 0.0, 0, 0, 0, 0
    for lo, hi in chunks(m):
        xc = cols64(x[lo:hi]) / 255.0
        pre = torch.einsum('ck,bkp->bcp', w64, xc) + b.double()[None, :, None]
        ref = torch.relu(pre)
        bound = (2.0 ** -11 + 48 * U) * torch.einsum('ck,bkp->bcp', wt, xc) + 2 * U * ref.abs() \
            + 2 * U * b.double().abs()[None, :, None] + 1e-30
        err = (y[lo:hi].view(hi - lo, 32, 400).double() - ref).abs()
        fwd_frac = max(fwd_frac, float((err / bound).max()))
        dz = (dy[lo:hi] * (y[lo:hi] > 0)).double().view(hi - lo, 32, 400)
        dw64 = dw64 + torch.einsum('bcp,bkp->ck', dz, xc)
        dwabs = dwabs + torch.einsum('bcp,bkp->ck', dz.abs(), xc)
        db64 = db64 + dz.sum((0, 2))
        dbabs = dbabs + dz.abs().sum((0, 2))
    ctas = min(m, WG_CTAS)
    per_cta = -(-m // ctas)
    reduce_terms = -(-ctas // 32) + 16
    bw = (2.0 ** -11 + (50 * per_cta + reduce_terms) * U) * dwabs + 1e-30
    bb = (16 * per_cta + reduce_terms) * U * dbabs + 1e-30
    dw_frac = float(((dw.double() - dw64).abs() / bw).max())
    db_frac = float(((db.double() - db64).abs() / bb).max())
    print(f'm={m} stride={stride}: observed / bound  y {fwd_frac:.3f}  dW {dw_frac:.3f}  db {db_frac:.3f}', flush=True)
    assert fwd_frac <= 1.0 and dw_frac <= 1.0 and db_frac <= 1.0
    return x, w, b, y, dy


@pytest.mark.parametrize('stride', [ROW, 30016])
def test_general_sizes_vs_fp64(stride):
    for m in general_sizes():
        check_general(m, stride, seed=m % 97)


def test_c4_minibatch_vs_fp64():
    """The C4 training minibatch: 131 072 rows."""
    check_general(131072, ROW, seed=5)


# ---- 3. determinism, capture, refusals --------------------------------------------------------------------------------
def test_deterministic_eager_and_graph():
    m = 4096
    w, b = orthogonal_weights(1)
    x = frames(m, ROW, 1)
    y1, y2 = forward(x, w, b), forward(x, w, b)
    assert torch.equal(y1, y2)
    dy = torch.randn(m, 32, 20, 20, device='cuda')
    d1, d2 = wgrad(x, y1, dy), wgrad(x, y1, dy)
    assert torch.equal(d1[0], d2[0]) and torch.equal(d1[1], d2[1])
    yg = torch.empty_like(y1)
    dwg, dbg = torch.empty(32, 256, device='cuda'), torch.empty(32, device='cuda')
    ws = torch.empty(lib().pb_conv1_u8_wgrad_workspace_bytes(m), dtype=torch.uint8, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            sp = _native.stream_ptr(s)
            _native.check(lib().pb_conv1_u8_forward(_native.ptr(x), ROW, m, _native.ptr(w), _native.ptr(b),
                                                    _native.ptr(yg), sp))
            _native.check(lib().pb_conv1_u8_wgrad(_native.ptr(x), ROW, m, _native.ptr(yg), _native.ptr(dy),
                                                  _native.ptr(dwg), _native.ptr(dbg), _native.ptr(ws), ws.numel(), sp))
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        yg.zero_(), dwg.zero_(), dbg.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, y1) and torch.equal(dwg, d1[0]) and torch.equal(dbg, d1[1])


def test_refusals_launch_nothing():
    L = lib()
    m = 8
    x = frames(m, ROW, 0)
    w, b = orthogonal_weights(0)
    y = torch.empty(m, 32, 20, 20, device='cuda')
    dw, db = torch.empty(32, 256, device='cuda'), torch.empty(32, device='cuda')
    nws = L.pb_conv1_u8_wgrad_workspace_bytes(m)
    ws = torch.empty(nws + 16, dtype=torch.uint8, device='cuda')
    P, sp = _native.ptr, _native.stream_ptr()
    xp = x.data_ptr()
    fwd_bad = [(C.c_void_p(0), ROW, P(w), P(b), P(y)), (C.c_void_p(xp + 1), ROW, P(w), P(b), P(y)),
               (P(x), ROW - 16, P(w), P(b), P(y)), (P(x), ROW + 8, P(w), P(b), P(y)), (P(x), ROW, None, P(b), P(y)),
               (P(x), ROW, C.c_void_p(w.data_ptr() + 4), P(b), P(y)), (P(x), ROW, P(w), None, P(y)),
               (P(x), ROW, P(w), P(b), C.c_void_p(y.data_ptr() + 4))]
    wg_bad = [(C.c_void_p(0), ROW, P(y), P(y), P(dw), P(db), P(ws), nws), (P(x), ROW + 4, P(y), P(y), P(dw), P(db), P(ws), nws),
              (P(x), ROW, C.c_void_p(y.data_ptr() + 4), P(y), P(dw), P(db), P(ws), nws),
              (P(x), ROW, P(y), None, P(dw), P(db), P(ws), nws), (P(x), ROW, P(y), P(y), None, P(db), P(ws), nws),
              (P(x), ROW, P(y), P(y), P(dw), None, P(ws), nws), (P(x), ROW, P(y), P(y), P(dw), P(db), None, nws),
              (P(x), ROW, P(y), P(y), P(dw), P(db), P(ws), nws - 4),
              (P(x), ROW, P(y), P(y), P(dw), P(db), C.c_void_p(ws.data_ptr() + 4), nws)]
    before = L.pb_launch_count()
    for a in fwd_bad:
        assert L.pb_conv1_u8_forward(a[0], a[1], m, a[2], a[3], a[4], sp) == _native.PB_ERR_INVALID, a
    for a in wg_bad:
        assert L.pb_conv1_u8_wgrad(a[0], a[1], m, *a[2:], sp) == _native.PB_ERR_INVALID, a
    with pytest.raises(APIUsageError):
        _native.check(L.pb_conv1_u8_forward(P(x), ROW, -1, P(w), P(b), P(y), sp))
    assert L.pb_conv1_u8_forward(P(x), ROW, 0, P(w), P(b), P(y), sp) == _native.PB_OK
    assert L.pb_conv1_u8_wgrad(P(x), ROW, 0, P(y), P(y), P(dw), P(db), P(ws), 16, sp) == _native.PB_OK
    assert L.pb_launch_count() == before


# ---- 4. model level ---------------------------------------------------------------------------------------------------
def pong_env():
    from test_gpu_policy_lstm import fake_env
    return fake_env((4, 84, 84), 6, np.uint8)


def model_pair(seed, **kw):
    torch.manual_seed(seed)
    a = models.Convolutional(pong_env(), **kw).cuda()
    b_ = models.Convolutional(pong_env(), **kw).cuda()
    b_.load_state_dict(a.state_dict())
    b_.fast_path = False
    return a, b_


def propagated_bound(model, x, c=4):
    """Elementwise bound on |out - out64| for the fast path's logits and values, by layer in fp64: conv1's bound (the
    module docstring, at the fp64 activations), then for each later layer (W, b, K terms per output, the layers run in
    fp32: fp32_library_math) e_out = |W| * e_in + c * K * 2^-24 * (|W| * (|a| + e_in) + |b|), and relu is 1-Lipschitz.
    c = 4 leaves room for cuDNN's choice of algorithm (a Winograd transform sums more terms than the dot product)."""
    net = model.network
    a = x.double() / 255.0
    w1, b1 = net[0].weight.double(), net[0].bias.double()
    a1 = torch.relu(F.conv2d(a, w1, b1, stride=4))
    e = (2.0 ** -11 + 48 * U) * F.conv2d(a, w1.abs(), stride=4) + 2 * U * a1.abs() + 2 * U * b1.abs()[None, :, None, None]
    a = a1

    def layer(a, e, fn, w, b_, k):
        pre = fn(a, w, b_)
        babs = fn(torch.zeros_like(a), torch.zeros_like(w), b_.abs())          # |b|, broadcast like the layer's bias
        e_out = fn(e, w.abs(), None) + c * k * U * (fn(a.abs() + e, w.abs(), None) + babs)
        return pre, e_out
    for conv in (net[2], net[4]):
        w, b_ = conv.weight.double(), conv.bias.double()
        k = w[0].numel()
        pre, e = layer(a, e, lambda t, w_, bb: F.conv2d(t, w_, bb, stride=conv.stride), w, b_, k)
        a = torch.relu(pre)
    a, e = a.flatten(1), e.flatten(1)
    fc = net[7]
    pre, e = layer(a, e, F.linear, fc.weight.double(), fc.bias.double(), fc.in_features)
    a = torch.relu(pre)
    outs = []
    for head in (model.actor, model.value_fn):
        outs.append(layer(a, e, F.linear, head.weight.double(), head.bias.double(), head.in_features))
    return outs


def test_model_forward_fast_vs_fp64(monkeypatch):
    """logits and values of the fast path against an fp64 restatement of the model, elementwise within
    propagated_bound (conv1's TF32 bound carried through the later layers plus their own fp32 rounding)."""
    fp32_library_math(monkeypatch)
    fast, stock = model_pair(0)
    x = frames(512, ROW, 3)
    calls = []
    orig = models._Conv1U8Function.apply
    monkeypatch.setattr(models._Conv1U8Function, 'apply', lambda *a: calls.append(1) or orig(*a))
    with torch.no_grad():
        lf, vf = fast(x)
        ls, vs = stock(x)
        (l64, bl), (v64, bv) = propagated_bound(stock, x)
    assert len(calls) == 1
    # all-0 frame rows with zero conv1 bias give exact zeros through every layer: bound and error both 0 there
    fl = float(((lf.double() - l64).abs() / (bl + 1e-30)).max())
    fv = float(((vf.double() - v64).abs() / (bv + 1e-30)).max())
    es = max(float((ls.double() - l64).abs().max()), float((vs.double() - v64).abs().max()))
    ef = max(float((lf.double() - l64).abs().max()), float((vf.double() - v64).abs().max()))
    print(f'model outputs vs fp64: fast {ef:.2e} (observed / bound: logits {fl:.3f}, values {fv:.3f}), '
          f'stock {es:.2e}', flush=True)
    assert fl <= 1.0 and fv <= 1.0


@pytest.mark.parametrize('case', ['channels_last', 'downsample', 'float_input', 'first_layer', 'strided_rows'])
def test_outside_fast_path_is_stock(case):
    kw = {'channels_last': dict(channels_last=True), 'downsample': dict(downsample=2, flat_size=64)}.get(case, {})
    fast, stock = model_pair(1, **kw)
    x = frames(64, ROW, 4).contiguous()
    if case == 'channels_last':
        x = x.permute(0, 2, 3, 1).contiguous()
    elif case == 'float_input':
        x = x.float()
    elif case == 'first_layer':
        for mdl in (fast, stock):
            old = mdl.network[0]
            mdl.network[0] = torch.nn.Conv2d(4, 32, 8, stride=4, bias=False).cuda()
            with torch.no_grad():
                mdl.network[0].weight.copy_(old.weight)
    elif case == 'strided_rows':
        x = frames(64, ROW + 8, 4)           # rows 8 bytes apart from 16-byte alignment: not the kernel's layout
    calls = []
    orig = models._Conv1U8Function.apply
    models._Conv1U8Function.apply = lambda *a: calls.append(1) or orig(*a)
    try:
        with torch.no_grad():
            a, b_ = fast(x), stock(x)
    finally:
        models._Conv1U8Function.apply = orig
    assert not calls
    assert torch.equal(a[0], b_[0]) and torch.equal(a[1], b_[1])


def fp32_library_math(monkeypatch):
    """cuDNN and cuBLAS in full fp32 for the layers both paths share: with TF32 there (torch's cuDNN default) their
    rounding, and the stock conv1's TF32 rounding of x / 255, hide the difference under test."""
    monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', False)
    monkeypatch.setattr(torch.backends.cuda.matmul, 'allow_tf32', False)


def test_model_minibatch_gradients_fast_vs_stock(monkeypatch):
    """Gradients of every parameter from one PPO minibatch (fused_ppo_loss) on pong frames: fast vs stock path within
    1.5e-2 of each tensor's largest gradient (the rule DESIGN.md §4 uses between update paths), the shared layers in
    fp32 (fp32_library_math)."""
    import pufferlib_b200
    fp32_library_math(monkeypatch)
    from pufferlib_b200 import clean_pufferl
    fast, stock = model_pair(2)
    m = 2048
    x = frames(m, ROW, 6)
    gen = torch.Generator(device='cuda').manual_seed(9)
    act = torch.randint(0, 6, (m,), device='cuda', generator=gen)
    old_lp = -torch.rand(m, device='cuda', generator=gen) - 1.0
    adv = torch.randn(m, device='cuda', generator=gen)
    ret, old_v = torch.randn(m, device='cuda', generator=gen), torch.randn(m, device='cuda', generator=gen)
    cfg = pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    grads = []
    for mdl in (fast, stock):
        logits, value = mdl(x)
        loss, _ = clean_pufferl.fused_ppo_loss(logits, value, act, old_lp, adv, ret, old_v, cfg)
        loss.backward()
        grads.append([p.grad.detach().clone() for p in mdl.parameters()])
    worst = 0.0
    for (name, _), gf, gs in zip(fast.named_parameters(), *grads):
        frac = float((gf - gs).abs().max() / gs.abs().max())
        worst = max(worst, frac)
        assert frac <= 1.5e-2, (name, frac)
    print(f'minibatch gradients: worst difference {worst:.2e} of the tensor maximum', flush=True)


# ---- 5. through the trainer -------------------------------------------------------------------------------------------
def test_pong_train_fast_vs_stock(monkeypatch):
    """train() on pong (256 envs x 32 steps, bptt 8, 2 minibatches, 2 epochs), same seed, same rollout (both trainers
    collect with the fast path, whose launches are deterministic), then train() with fast_path on vs off, the layers both
    share in fp32 (fp32_library_math): the plan ('model', 'gathered') in both, the fast trainer's train() through
    _Conv1U8Function and the stock one's not, losses within 1e-4 relative, and per parameter tensor (conv1's weight and
    bias among them) a median difference of at most 2e-6, at most 2 % of the elements more than 2e-5 apart and none more
    than the 4 optimizer steps' lr.  Observed: conv1's weight median 9.9e-7, 117 of 8 192 above 2e-5 (1.4 %), max 5.6e-4;
    the other tensors' medians are near 1e-8."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    from test_gpu_config_updates import ppo_config
    fp32_library_math(monkeypatch)
    n, h, bptt, nm = 256, 32, 8, 2
    lr = 2.5e-4
    plans, calls = [], []
    update_plan = clean_pufferl.update_plan
    monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(update_plan(d)) or plans[-1])
    orig = models._Conv1U8Function.apply
    monkeypatch.setattr(models._Conv1U8Function, 'apply', lambda *a: calls.append(1) or orig(*a))
    res = {}
    for fast in (True, False):
        vec = pvec.make(ocean.env_creator('pong'), num_envs=n, backend=pvec.B200)
        torch.manual_seed(0)
        pol = cleanrl.Policy(models.Convolutional(vec.driver_env), fused_sample=True, seed=3).cuda()
        data = clean_pufferl.create(ppo_config('pong', n, h, bptt, nm, fused_loss=True, learning_rate=lr), vec, pol)
        clean_pufferl.evaluate(data)
        roll = {k: data.experience.__getattribute__(k).detach().cpu().numpy().copy()
                for k in ('obs', 'actions', 'logprobs', 'values')}
        pol.policy.fast_path = fast
        calls.clear()
        clean_pufferl.train(data)
        # 2 epochs x 2 minibatches, one call each on the fast path
        assert len(calls) == (4 if fast else 0), (fast, len(calls))
        assert (plans[-1].engine, plans[-1].form) == ('model', 'gathered'), plans[-1]
        losses = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy, data.losses.approx_kl,
                           data.losses.clipfrac, data.losses.explained_variance])
        res[fast] = (roll, dict((k, p.detach().clone()) for k, p in pol.policy.named_parameters()), losses)
        clean_pufferl.close(data)
    for k in res[True][0]:
        assert np.array_equal(res[True][0][k], res[False][0][k]), k
    print(f'losses fast {res[True][2]} stock {res[False][2]}', flush=True)
    assert np.allclose(res[True][2], res[False][2], rtol=1e-4, atol=1e-6)
    # the only difference between the two updates is conv1's TF32 operands on the fast path (W and dz rounded, 2^-11).
    # It reaches conv1's weight gradient most (1.45e-2 of its maximum in test_model_minibatch_gradients_fast_vs_stock:
    # dW sums 800 000 products of either sign), and Adam divides by sqrt(v), so conv1 weights whose gradient is within
    # that difference move apart by a fraction of a step (at most lr each); the bulk of every tensor stays within 2e-5
    for name, p in res[True][1].items():
        d = (p - res[False][1][name]).abs().double().flatten()
        above = int((d > 2e-5).sum())
        print(f'{name:24s} {d.numel():8d} elements: max {float(d.max()):.2e} median {float(d.median()):.2e} '
              f'{above} above 2e-5', flush=True)
        assert float(d.median()) <= 2e-6, name
        assert above <= d.numel() // 50, name
        assert float(d.max()) <= 4 * lr, name


def c4_budget(n, h, mb):
    """Peak device memory allowed for C4 on the fast path: the rollout observations and b_obs (n * h rows of 28 224
    bytes each), conv1's saved y1 and its gradient (2 * 12 800 floats per minibatch row), the other layers' saved
    activations and gradients (3 * (5184 + 3136 + 512) floats per row: conv2, conv3, the 512-unit Linear), plus 4 GiB
    for the per-row rollout tensors, parameters, optimizer state, cuDNN workspaces and the allocator.  A float copy of the
    minibatch frames (x / 255: 28 224 floats per row, 14.8 GB at C4) does not fit in it."""
    frames_ = 2 * n * h * ROW
    acts = mb * 4 * (2 * Y_ROW + 3 * (5184 + 3136 + 512))
    return frames_ + acts + 4 * 2 ** 30


def test_pong_c4_full_size_graphed():
    """C4 at full size: 4 096 envs x 128 steps, 4 minibatches of 131 072 rows, cuda_graph=True, two evaluate() + train()
    iterations through run_config (the first 16 envs replayed bit-exactly through the oracle, GAE against the oracle,
    finite losses, parameters moved), conv1 on the fast path, peak memory under c4_budget."""
    from test_gpu_configs import run_config
    n, h, nm = 4096, 128, 4
    calls = []
    orig = models._Conv1U8Function.apply
    models._Conv1U8Function.apply = lambda *a: calls.append(1) or orig(*a)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    try:
        data = run_config('pong', n, h, 16, nm, cuda_graph=True, iterations=2, replay_envs=16)
    finally:
        models._Conv1U8Function.apply = orig
    peak = torch.cuda.max_memory_allocated()
    budget = c4_budget(n, h, n * h // nm)
    print(f'C4 peak {peak / 2 ** 30:.2f} GiB, budget {budget / 2 ** 30:.2f} GiB, conv1 fast-path calls {len(calls)}, '
          f'graph replays {data.graph_replays}, train graph state {data.train_graph_state}', flush=True)
    assert calls and data.graph_replays >= 1 and data.train_graph_state == 2
    assert peak <= budget
