"""models.Convolutional's conv2 and conv3 on hand-written TF32 kernels (csrc/nature_trunk.cu): pb_nature_conv_forward,
pb_nature_conv_dgrad and pb_nature_conv_wgrad against exact restatements and fp64, their canaries, determinism, capture
and ABI refusals; the model's trunk path against the path with the trunk refused; train() on pong with it; C4 at full size
on pong and breakout_pixels.

Bounds (U = 2^-24, T = 2^-11 the TF32 cvt.rna unit).  Both operands of every product are rounded to TF32, so a product
is off by at most (2T + T^2) of its magnitude; the fp32 sums then add at most (n + 2) U of the sum of magnitudes for n
accumulating additions (taken sequential, the worst case of any order).
  forward  |y - y64| <= (2T + T^2 + (K + 2) U) conv(|x|, |w|) + 2 U (|y64| + |b|)   (bias add; relu is 1-Lipschitz)
  dgrad    |dx - dx64| <= (2T + T^2 + (K + 2) U) conv_transpose(|dz|, |w|)
  wgrad    |dW - dW64| <= (2T + T^2 + (R P8 + ceil(G / 32) + 16) U) sum |dz| |x_col|, R rows per CTA, P8 the pixels
           padded to 8, G CTAs; db: (R + ceil(G / 32) + 16) U sum |dz| (lane sums, shuffle tree, per-row adds, reduce).
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pufferlib_b200 import _native, models

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
T = 2.0 ** -11
WG_CTAS = 132
# layer: (C_in, H, KS, stride, P)
GEOM = {2: (32, 20, 4, 2, 81), 3: (64, 9, 3, 1, 49)}


def lib():
    return _native.lib()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def xshape(layer):
    cin, h = GEOM[layer][:2]
    return (cin, h, h)


def yshape(layer):
    ho = int(GEOM[layer][4] ** 0.5)
    return (64, ho, ho)


def padded(m, shape, fill, extra=2):
    """m rows of `shape` followed by `extra` rows of `fill` (never to be read, or canaries)."""
    buf = torch.full((m + extra,) + shape, fill, dtype=torch.float32, device='cuda')
    return buf, buf[:m]


def forward(layer, x, w, b):
    m = x.shape[0]
    yb, y = padded(m, yshape(layer), -7.0)
    _native.check(lib().pb_nature_conv_forward(layer, _native.ptr(x), m, _native.ptr(w), _native.ptr(b), _native.ptr(y),
                                               _native.stream_ptr()))
    assert bool((yb[m:] == -7.0).all()), 'rows after y were written'
    return y


def dgrad(layer, y, dy, w):
    m = y.shape[0]
    dxb, dx = padded(m, xshape(layer), -7.0)
    _native.check(lib().pb_nature_conv_dgrad(layer, _native.ptr(y), _native.ptr(dy), _native.ptr(w), m, _native.ptr(dx),
                                             _native.stream_ptr()))
    assert bool((dxb[m:] == -7.0).all()), 'rows after dx were written'
    return dx


def wgrad(layer, x, y, dy):
    m = x.shape[0]
    cin, _, ks = GEOM[layer][:3]
    dwb = torch.full((64 * cin * ks * ks + 16,), -7.0, device='cuda')
    dbb = torch.full((64 + 16,), -7.0, device='cuda')
    n = lib().pb_nature_conv_wgrad_workspace_bytes(layer, m)
    ws = torch.full((n + 64,), 0xA5, dtype=torch.uint8, device='cuda')
    _native.check(lib().pb_nature_conv_wgrad(layer, _native.ptr(x), _native.ptr(y), _native.ptr(dy), m, _native.ptr(dwb),
                                             _native.ptr(dbb), _native.ptr(ws), n, _native.stream_ptr()))
    assert bool((dwb[-16:] == -7.0).all()) and bool((dbb[-16:] == -7.0).all()), 'past dw / db written'
    assert bool((ws[n:] == 0xA5).all()), 'past the workspace written'
    return dwb[:-16].view(64, cin, ks, ks), dbb[:64]


def inputs(layer, m, seed, grid=False):
    """x (NaN rows after it), w, b, dy (NaN rows after it).  grid: every value on a coarse power-of-two grid (x in
    {0, .25, .., 1.75} with zeros, w and b multiples of 2^-6 in [-1/8, 1/8], dy multiples of 2^-4 in [-1/2, 1/2])."""
    cin, h, ks, s, _ = GEOM[layer]
    gen = torch.Generator(device='cuda').manual_seed(seed)
    xb, x = padded(m, xshape(layer), float('nan'))
    dyb, dy = padded(m, yshape(layer), float('nan'))
    if grid:
        x.copy_(torch.randint(-3, 8, x.shape, generator=gen, device='cuda').clamp_(min=0).float() / 4)
        w = torch.randint(-8, 9, (64, cin, ks, ks), generator=gen, device='cuda').float() / 64
        b = torch.randint(-8, 9, (64,), generator=gen, device='cuda').float() / 64
        dy.copy_(torch.randint(-8, 9, dy.shape, generator=gen, device='cuda').float() / 16)
    else:
        x.copy_(torch.relu(torch.randn(x.shape, generator=gen, device='cuda')))
        conv = torch.nn.Conv2d(cin, 64, ks, stride=s)
        torch.manual_seed(seed)
        models.layer_init(conv)
        w = conv.weight.detach().cuda().contiguous()
        b = (torch.rand(64, generator=gen, device='cuda') - 0.5) * 0.2
        dy.copy_(torch.randn(dy.shape, generator=gen, device='cuda'))
    if m > 2:
        x[0] = 0.0                      # an all-zero row: y = relu(b), dz masked where b <= 0
    return x, w, b, dy


def chunks(m, size=4096):
    return [(lo, min(m, lo + size)) for lo in range(0, m, size)]


# ---- 1. exact case ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('layer', [2, 3])
@pytest.mark.parametrize('m', [1, 3, 37])
def test_exact_bitwise(layer, m):
    """On the grids of `inputs(grid=True)` every operand is a TF32 value and every partial sum is a multiple of 2^-10
    (forward, dgrad) or 2^-6 (wgrad) far below 2^24 of that unit: every result is exact, so it must equal the fp64
    result rounded to fp32 bit for bit, in all three modes."""
    s = GEOM[layer][3]
    x, w, b, dy = inputs(layer, m, seed=m + layer, grid=True)
    y = forward(layer, x, w, b)
    assert torch.equal(y, torch.relu(F.conv2d(x.double(), w.double(), b.double(), stride=s)).float())
    dz = (dy * (y > 0)).double()
    dx = dgrad(layer, y, dy, w)
    assert torch.equal(dx, torch.nn.grad.conv2d_input(x.shape, w.double(), dz, stride=s).float())
    dw, db = wgrad(layer, x, y, dy)
    assert torch.equal(dw, torch.nn.grad.conv2d_weight(x.double(), w.shape, dz, stride=s).float())
    assert torch.equal(db, dz.sum((0, 2, 3)).float())


# ---- 2. general case against fp64 -------------------------------------------------------------------------------------
def check_general(layer, m, seed, zero_pre=False, scale=1.0):
    cin, h, ks, s, p = GEOM[layer]
    k = cin * ks * ks
    x, w, b, dy = inputs(layer, m, seed)
    if scale != 1.0:
        x.mul_(scale)
    if zero_pre:                        # every pre-activation exactly 0: y = relu(0) = 0 and the y > 0 mask drops all dz
        b = torch.zeros_like(b)
        x[:, :, :, :] = torch.where(torch.arange(cin, device='cuda')[None, :, None, None] % 2 == 0, x, 0.0)
        w = w.clone()
        w[:, 0::2] = 0.0                # each product has a zero factor
    y = forward(layer, x, w, b)
    dx = dgrad(layer, y, dy, w)
    dw, db = wgrad(layer, x, y, dy)
    w64, wa = w.double(), w.double().abs()
    fwd, dgr = 0.0, 0.0
    dw64 = dwa = db64 = dba = 0
    for lo, hi in chunks(m):
        x64 = x[lo:hi].double()
        ref = torch.relu(F.conv2d(x64, w64, b.double(), stride=s))
        bound = (2 * T + T * T + (k + 2) * U) * F.conv2d(x64.abs(), wa, stride=s) \
            + 2 * U * (ref.abs() + b.double().abs()[None, :, None, None]) + 1e-300
        fwd = max(fwd, float(((y[lo:hi].double() - ref).abs() / bound).max()))
        dz = (dy[lo:hi] * (y[lo:hi] > 0)).double()
        ref = torch.nn.grad.conv2d_input(x64.shape, w64, dz, stride=s)
        kd = 64 * (ks // s) ** 2
        bound = (2 * T + T * T + (kd + 2) * U) * torch.nn.grad.conv2d_input(x64.shape, wa, dz.abs(), stride=s) + 1e-300
        dgr = max(dgr, float(((dx[lo:hi].double() - ref).abs() / bound).max()))
        dw64 = dw64 + torch.nn.grad.conv2d_weight(x64, w.shape, dz, stride=s)
        dwa = dwa + torch.nn.grad.conv2d_weight(x64.abs(), w.shape, dz.abs(), stride=s)
        db64 = db64 + dz.sum((0, 2, 3))
        dba = dba + dz.abs().sum((0, 2, 3))
    ctas = min(m, WG_CTAS)
    rows = -(-m // ctas)
    red = -(-ctas // 32) + 16
    bw = (2 * T + T * T + (rows * ((p + 7) // 8 * 8) + red) * U) * dwa + 1e-300
    bb = (rows + red) * U * dba + 1e-300
    wg = float(((dw.double() - dw64).abs() / bw).max())
    dbf = float(((db.double() - db64).abs() / bb).max())
    print(f'layer {layer} m={m}: observed / bound  y {fwd:.3f}  dx {dgr:.3f}  dW {wg:.3f}  db {dbf:.3f}', flush=True)
    assert fwd <= 1.0 and dgr <= 1.0 and wg <= 1.0 and dbf <= 1.0
    return y


def general_sizes():
    g = sms()
    return sorted({1, 2, g - 1, g, g + 1, 2 * g + 1, WG_CTAS - 1, WG_CTAS + 1, 2 * WG_CTAS + 1, 4096})


@pytest.mark.parametrize('layer', [2, 3])
def test_general_sizes_vs_fp64(layer):
    for m in general_sizes():
        check_general(layer, m, seed=m % 89)


@pytest.mark.parametrize('layer', [2, 3])
def test_c4_minibatch_vs_fp64(layer):
    """The C4 training minibatch: 131 072 rows."""
    check_general(layer, 131072, seed=5)


@pytest.mark.parametrize('layer', [2, 3])
def test_zero_preactivations_and_large_inputs(layer):
    y = check_general(layer, 37, seed=11, zero_pre=True)
    assert bool((y == 0).all())        # relu(0) = 0: the mask drops every dz, so dx, dW and db must be 0 (checked above)
    check_general(layer, 37, seed=12, scale=2.0 ** 40)


# ---- 3. determinism, capture, refusals --------------------------------------------------------------------------------
@pytest.mark.parametrize('layer', [2, 3])
def test_deterministic_eager_and_graph(layer):
    m = 4096
    x, w, b, dy = inputs(layer, m, 1)
    y1, y2 = forward(layer, x, w, b), forward(layer, x, w, b)
    assert torch.equal(y1, y2)
    dx1, dx2 = dgrad(layer, y1, dy, w), dgrad(layer, y1, dy, w)
    assert torch.equal(dx1, dx2)
    (a1, c1), (a2, c2) = wgrad(layer, x, y1, dy), wgrad(layer, x, y1, dy)
    assert torch.equal(a1, a2) and torch.equal(c1, c2)
    yg, dxg, dwg, dbg = torch.empty_like(y1), torch.empty_like(dx1), torch.empty_like(a1), torch.empty_like(c1)
    ws = torch.empty(lib().pb_nature_conv_wgrad_workspace_bytes(layer, m), dtype=torch.uint8, device='cuda')
    P = _native.ptr
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            sp = _native.stream_ptr(s)
            _native.check(lib().pb_nature_conv_forward(layer, P(x), m, P(w), P(b), P(yg), sp))
            _native.check(lib().pb_nature_conv_dgrad(layer, P(yg), P(dy), P(w), m, P(dxg), sp))
            _native.check(lib().pb_nature_conv_wgrad(layer, P(x), P(yg), P(dy), m, P(dwg), P(dbg), P(ws), ws.numel(), sp))
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        for t_ in (yg, dxg, dwg, dbg):
            t_.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, y1) and torch.equal(dxg, dx1) and torch.equal(dwg, a1) and torch.equal(dbg, c1)


def test_refusals_launch_nothing():
    L = lib()
    P, sp, m = _native.ptr, _native.stream_ptr(), 8
    x, w, b, dy = inputs(3, m, 0)
    y, dx = torch.empty(m, 64, 7, 7, device='cuda'), torch.empty_like(x)
    dw, db = torch.empty_like(w), torch.empty(64, device='cuda')
    nws = L.pb_nature_conv_wgrad_workspace_bytes(3, m)
    ws = torch.empty(nws + 16, dtype=torch.uint8, device='cuda')
    off = lambda t_, k: C.c_void_p(t_.data_ptr() + k)  # noqa: E731
    assert L.pb_nature_conv_wgrad_workspace_bytes(4, m) == 0
    before = L.pb_launch_count()
    for layer in (1, 4, 0, -2):
        assert L.pb_nature_conv_forward(layer, P(x), m, P(w), P(b), P(y), sp) == _native.PB_ERR_INVALID
        assert L.pb_nature_conv_dgrad(layer, P(y), P(dy), P(w), m, P(dx), sp) == _native.PB_ERR_INVALID
        assert L.pb_nature_conv_wgrad(layer, P(x), P(y), P(dy), m, P(dw), P(db), P(ws), nws, sp) == _native.PB_ERR_INVALID
    fwd_bad = [(None, P(w), P(b), P(y)), (off(x, 4), P(w), P(b), P(y)), (P(x), None, P(b), P(y)),
               (P(x), off(w, 8), P(b), P(y)), (P(x), P(w), None, P(y)), (P(x), P(w), off(b, 2), P(y)),
               (P(x), P(w), P(b), None), (P(x), P(w), P(b), off(y, 4))]
    for a in fwd_bad:
        assert L.pb_nature_conv_forward(3, a[0], m, a[1], a[2], a[3], sp) == _native.PB_ERR_INVALID, a
    assert L.pb_nature_conv_forward(3, P(x), -1, P(w), P(b), P(y), sp) == _native.PB_ERR_INVALID
    dg_bad = [(None, P(dy), P(w), P(dx)), (off(y, 4), P(dy), P(w), P(dx)), (P(y), off(dy, 8), P(w), P(dx)),
              (P(y), P(dy), None, P(dx)), (P(y), P(dy), off(w, 4), P(dx)), (P(y), P(dy), P(w), off(dx, 12))]
    for a in dg_bad:
        assert L.pb_nature_conv_dgrad(3, a[0], a[1], a[2], m, a[3], sp) == _native.PB_ERR_INVALID, a
    wg_bad = [(None, P(y), P(dy), P(dw), P(db), P(ws), nws), (off(x, 4), P(y), P(dy), P(dw), P(db), P(ws), nws),
              (P(x), off(y, 4), P(dy), P(dw), P(db), P(ws), nws), (P(x), P(y), None, P(dw), P(db), P(ws), nws),
              (P(x), P(y), P(dy), off(dw, 2), P(db), P(ws), nws), (P(x), P(y), P(dy), P(dw), None, P(ws), nws),
              (P(x), P(y), P(dy), P(dw), P(db), None, nws), (P(x), P(y), P(dy), P(dw), P(db), off(ws, 4), nws),
              (P(x), P(y), P(dy), P(dw), P(db), P(ws), nws - 4)]
    for a in wg_bad:
        assert L.pb_nature_conv_wgrad(3, a[0], a[1], a[2], m, *a[3:], sp) == _native.PB_ERR_INVALID, a
    for layer in (2, 3):
        assert L.pb_nature_conv_forward(layer, P(x), 0, P(w), P(b), P(y), sp) == _native.PB_OK
        assert L.pb_nature_conv_dgrad(layer, P(y), P(dy), P(w), 0, P(dx), sp) == _native.PB_OK
        assert L.pb_nature_conv_wgrad(layer, P(x), P(y), P(dy), 0, P(dw), P(db), P(ws), 16, sp) == _native.PB_OK
    assert L.pb_launch_count() == before


# ---- 4. model level ---------------------------------------------------------------------------------------------------
def pong_env():
    from test_gpu_policy_lstm import fake_env
    return fake_env((4, 84, 84), 6, np.uint8)


def frames(m, seed):
    from test_gpu_nature_conv1 import ROW, frames as f
    return f(m, ROW, seed)


def count_calls(monkeypatch):
    calls = []
    orig = models._ConvReLUTF32Function.apply
    monkeypatch.setattr(models._ConvReLUTF32Function, 'apply', lambda *a: calls.append(a[-1]) or orig(*a))
    return calls


def refuse_trunk(model):
    """The same model with the trunk refused: conv1 on its kernel, network[2:] on cuDNN (today's path)."""
    model._trunk_ok = lambda: False
    return model


def model_pair(seed):
    torch.manual_seed(seed)
    a = models.Convolutional(pong_env()).cuda()
    b_ = models.Convolutional(pong_env()).cuda()
    b_.load_state_dict(a.state_dict())
    return a, refuse_trunk(b_)


def test_model_forward_vs_fp64(monkeypatch):
    """logits and values on the trunk path against an fp64 restatement, elementwise within propagated_bound with TF32
    terms for conv1 (its own bound) and for conv2, conv3 (2T + T^2 per product on top of the fp32 terms), the Linear
    and the heads in fp32."""
    from test_gpu_nature_conv1 import propagated_bound
    monkeypatch.setattr(torch.backends.cuda.matmul, 'allow_tf32', False)
    calls = count_calls(monkeypatch)
    model, _ = model_pair(0)
    x = frames(512, 3)
    with torch.no_grad():
        lf, vf = model(x)
        # the bound's per-layer term c K U must cover 2T + T^2 + (K + 2) U for K = 512: c = 40 does (c K U = 1.22e-3)
        (l64, bl), (v64, bv) = propagated_bound(model, x, c=40)
    assert calls == [2, 3]
    fl = float(((lf.double() - l64).abs() / (bl + 1e-30)).max())
    fv = float(((vf.double() - v64).abs() / (bv + 1e-30)).max())
    print(f'model outputs vs fp64, observed / bound: logits {fl:.3f}, values {fv:.3f}', flush=True)
    assert fl <= 1.0 and fv <= 1.0


CASES = ['tf32_off', 'fast_path_off', 'float_input', 'conv2_no_bias', 'conv3_no_bias', 'conv3_reflect', 'conv2_dilated',
         'relu_swapped', 'conv3_strided_weight']


@pytest.mark.parametrize('case', CASES)
def test_outside_trunk_path_is_stock(case, monkeypatch):
    torch.manual_seed(1)
    a = models.Convolutional(pong_env()).cuda()
    if case == 'conv2_dilated':        # same output shape as the stock layer only with kernel 2: dilation 2 covers 3
        a.network[2] = torch.nn.Conv2d(32, 64, 2, stride=2, dilation=3).cuda()
    elif case in ('conv2_no_bias', 'conv3_no_bias'):
        i = 2 if case == 'conv2_no_bias' else 4
        old = a.network[i]
        a.network[i] = torch.nn.Conv2d(old.in_channels, 64, old.kernel_size, stride=old.stride, bias=False).cuda()
        with torch.no_grad():
            a.network[i].weight.copy_(old.weight)
    elif case == 'conv3_reflect':
        a.network[4].padding_mode = 'reflect'
    elif case == 'relu_swapped':
        a.network[3] = torch.nn.LeakyReLU(0.0)
    elif case == 'conv3_strided_weight':
        a.network[4].weight.data = a.network[4].weight.data.transpose(0, 1).contiguous().transpose(0, 1)
    b_ = models.Convolutional(pong_env()).cuda()
    b_.network = a.network
    b_.load_state_dict(a.state_dict())
    refuse_trunk(b_)
    x = frames(64, 4).contiguous()
    if case == 'tf32_off':
        monkeypatch.setattr(torch.backends.cudnn, 'allow_tf32', False)
    elif case == 'fast_path_off':
        a.fast_path = b_.fast_path = False
    elif case == 'float_input':
        x = x.float()
    calls = count_calls(monkeypatch)
    with torch.no_grad():
        ra, rb = a(x), b_(x)
    assert not calls
    assert torch.equal(ra[0], rb[0]) and torch.equal(ra[1], rb[1])


def minibatch(m, seed):
    import pufferlib_b200
    x = frames(m, seed)
    gen = torch.Generator(device='cuda').manual_seed(seed + 3)
    act = torch.randint(0, 6, (m,), device='cuda', generator=gen)
    old_lp = -torch.rand(m, device='cuda', generator=gen) - 1.0
    adv = torch.randn(m, device='cuda', generator=gen)
    ret, old_v = torch.randn(m, device='cuda', generator=gen), torch.randn(m, device='cuda', generator=gen)
    cfg = pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    return x, (act, old_lp, adv, ret, old_v, cfg)


def test_model_minibatch_gradients_vs_refused(monkeypatch):
    """Gradients of every parameter from one PPO minibatch on pong frames, allow_tf32 on: trunk path vs the trunk
    refused (cuDNN TF32) within 1.5e-2 of each tensor's largest gradient (the rule DESIGN.md §4 uses between update
    paths)."""
    from pufferlib_b200 import clean_pufferl
    calls = count_calls(monkeypatch)
    new, old = model_pair(2)
    x, args = minibatch(2048, 6)
    grads = []
    for mdl in (new, old):
        logits, value = mdl(x)
        loss, _ = clean_pufferl.fused_ppo_loss(logits, value, *args)
        loss.backward()
        grads.append([p.grad.detach().clone() for p in mdl.parameters()])
    assert calls == [2, 3]
    worst = 0.0
    for (name, _), gn, go in zip(new.named_parameters(), *grads):
        frac = float((gn - go).abs().max() / go.abs().max())
        worst = max(worst, frac)
        assert frac <= 1.5e-2, (name, frac)
    print(f'minibatch gradients: worst difference {worst:.2e} of the tensor maximum', flush=True)


# ---- 5. through the trainer -------------------------------------------------------------------------------------------
def test_pong_train_vs_refused(monkeypatch):
    """train() on pong (256 envs x 32 steps, bptt 8, 2 minibatches, 2 epochs), same rollout (both trainers collect with
    the trunk refused), then train() with the trunk path vs refused, allow_tf32 on in both: plan ('model', 'gathered'),
    the new Function twice per minibatch, losses within 2e-3 relative (both paths round conv2 / conv3 to TF32, each
    differently: 2T relative per product), and per parameter tensor a median difference of at most lr / 10 and a maximum
    of at most 8 lr (each of the 4 Adam steps moves an element by about lr at most in each trainer)."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    from test_gpu_config_updates import ppo_config
    n, h, bptt, nm = 256, 32, 8, 2
    lr = 2.5e-4
    plans = []
    update_plan = clean_pufferl.update_plan
    monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(update_plan(d)) or plans[-1])
    calls = count_calls(monkeypatch)
    res = {}
    for trunk in (True, False):
        vec = pvec.make(ocean.env_creator('pong'), num_envs=n, backend=pvec.B200)
        torch.manual_seed(0)
        net = models.Convolutional(vec.driver_env)
        pol = cleanrl.Policy(net, fused_sample=True, seed=3).cuda()
        data = clean_pufferl.create(ppo_config('pong', n, h, bptt, nm, fused_loss=True, learning_rate=lr), vec, pol)
        net._trunk_ok = lambda: False
        clean_pufferl.evaluate(data)
        roll = {k: getattr(data.experience, k).detach().cpu().numpy().copy() for k in ('obs', 'actions', 'logprobs', 'values')}
        if trunk:
            del net._trunk_ok
        calls.clear()
        clean_pufferl.train(data)
        assert len(calls) == (8 if trunk else 0), (trunk, len(calls))
        assert (plans[-1].engine, plans[-1].form) == ('model', 'gathered'), plans[-1]
        losses = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy, data.losses.approx_kl,
                           data.losses.clipfrac, data.losses.explained_variance])
        res[trunk] = (roll, dict((k, p.detach().clone()) for k, p in pol.policy.named_parameters()), losses)
        clean_pufferl.close(data)
    for k in res[True][0]:
        assert np.array_equal(res[True][0][k], res[False][0][k]), k
    print(f'losses trunk {res[True][2]} refused {res[False][2]}', flush=True)
    assert np.allclose(res[True][2], res[False][2], rtol=2e-3, atol=1e-5)
    for name, p in res[True][1].items():
        d = (p - res[False][1][name]).abs().double().flatten()
        print(f'{name:24s} {d.numel():8d} elements: max {float(d.max()):.2e} median {float(d.median()):.2e}', flush=True)
        assert float(d.median()) <= lr / 10, name
        assert float(d.max()) <= 8 * lr, name


@pytest.mark.parametrize('kind', ['pong', 'breakout_pixels'])
def test_c4_full_size_graphed(kind, monkeypatch):
    """C4 at full size: 4 096 envs x 128 steps, 4 minibatches of 131 072 rows, cuda_graph=True, two evaluate() +
    train() iterations: the trunk path taken, the update captured (train graph state 2), finite losses, peak memory
    under test_gpu_nature_conv1.c4_budget."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    from test_gpu_config_updates import ppo_config
    from test_gpu_nature_conv1 import c4_budget
    n, h, nm = 4096, 128, 4
    import gc
    calls = count_calls(monkeypatch)
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()             # whatever earlier tests in this process still hold
    vec = pvec.make(ocean.env_creator(kind), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Convolutional(vec.driver_env), fused_sample=True, seed=3).cuda()
    data = clean_pufferl.create(ppo_config(kind, n, h, 16, nm, cuda_graph=True), vec, pol)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        assert all(np.isfinite(v) for v in (data.losses.policy_loss, data.losses.value_loss, data.losses.entropy))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    budget = c4_budget(n, h, n * h // nm)
    print(f'{kind} C4 peak {peak / 2 ** 30:.2f} GiB, budget {budget / 2 ** 30:.2f} GiB, trunk calls {len(calls)}, '
          f'graph state {data.graph_state}, train graph state {data.train_graph_state}', flush=True)
    assert calls and data.train_graph_state == 2
    assert peak <= budget
    clean_pufferl.close(data)
