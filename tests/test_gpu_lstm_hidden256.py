"""LSTMWrapper(Default(hidden_size=256), input_size=256, hidden_size=256) on the fused recurrent kernels: the H = 256
instances of pb_policy_lstm_sample (csrc/policy_lstm.cu) and pb_lstm_bptt_forward / _backward (+ _rows,
csrc/lstm_bptt.cu), the H-generic packs of models.LSTMWrapper, and train()'s 'bptt' engine at that size.

The kernel outputs are checked against fp64 restatements of their TF32 operand rounding, as the H = 128 tests do
(test_gpu_policy_lstm.py, test_gpu_lstm_bptt.py); the forward at T = 1 against the rollout step bitwise; the gradients
against fp64 autograd; the segment-view entry points against the gathered ones bitwise; train() against the cuDNN path.
A CTA of the H = 256 kernels owns 64 rows, so the batch sizes sit on that tile's edges."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from test_gpu_lstm_bptt import keep_relu_off_zero, snapshot_train
from test_gpu_lstm_train_graph import adam_state, fp32_matmul, losses, segment_setup  # noqa: F401 (fixture)
from test_gpu_policy_lstm import fake_env, make_config, reference_step, rollout_oracle, sharpen
from util_gpu import off_boundary_mismatches, rna

gpu = pytest.mark.gpu
H = 256
TILE = 64               # rows (segments) per CTA of the H = 256 kernels
TOL = 2e-4              # per-step outputs vs fp64
TOL_SEQ = 5e-4          # after 16 recurrent steps
TOL_GRAD = 5e-3         # each gradient vs fp64 autograd, relative to its largest entry
P = _native.ptr
NAN = float('nan')


def cpu(x):
    return x.detach().cpu().numpy()


def make_net(feats, n_act, hidden=H, layers=1):
    torch.manual_seed(0)
    env = fake_env((feats,), n_act)
    net = models.LSTMWrapper(env, models.Default(env, hidden_size=hidden), input_size=hidden, hidden_size=hidden,
                             num_layers=layers)
    sharpen(net)
    return net.cuda()


def reference_forward(net, x, h0, c0):
    """fp64 restatement of pb_lstm_bptt_forward at any H (reference_step over the T steps) -> (out, h_T, c_T)."""
    bsz, steps, _ = x.shape
    hid = net.recurrent.hidden_size
    h = torch.zeros(bsz, hid, dtype=torch.float64, device='cuda') if h0 is None else h0.double()
    c = torch.zeros(bsz, hid, dtype=torch.float64, device='cuda') if c0 is None else c0.double()
    outs = []
    for t in range(steps):
        h, c, out = reference_step(net, x[:, t], h, c)
        outs.append(out)
    return torch.stack(outs, 1).reshape(bsz * steps, -1), h, c


def forward_kernel(net, x, h0=None, c0=None, guard=5, seg=None):
    """pb_lstm_bptt_forward on x [B, T, F] (or _rows on the segment view `seg` [E, G, T, F]) at the net's H ->
    (out, h_T, c_T, saved), NaN canaries past every output."""
    hid = net.recurrent.hidden_size
    if seg is not None:
        e_, g_, steps, feats = seg.shape
        bsz = e_ * g_
    else:
        bsz, steps, feats = x.shape
    m = bsz * steps
    n_act = net.policy.decoder.weight.shape[0]
    with torch.no_grad():
        w_enc, b_enc, w_gates, b_gates, w_cat, b_cat = net.fused_operands()
    out = torch.full((m + guard, w_cat.shape[0]), NAN, device='cuda')
    hT, cT = torch.full((bsz + guard, hid), NAN, device='cuda'), torch.full((bsz + guard, hid), NAN, device='cuda')
    saved = torch.full((m + guard, 8 * hid), NAN, device='cuda')
    lib = _native.lib()
    if seg is not None:
        _native.check(lib.pb_lstm_bptt_forward_rows(
            P(seg), feats, bsz, steps, g_, seg.stride(0), seg.stride(1), seg.stride(2), P(h0), P(c0), P(w_enc),
            P(b_enc), P(w_gates), P(b_gates), P(w_cat), P(b_cat), hid, hid, n_act, P(out), P(hT), P(cT), P(saved),
            _native.stream_ptr()))
    else:
        _native.check(lib.pb_lstm_bptt_forward(
            P(x), x.stride(1), feats, bsz, steps, P(h0), P(c0), P(w_enc), P(b_enc), P(w_gates), P(b_gates), P(w_cat),
            P(b_cat), hid, hid, n_act, P(out), P(hT), P(cT), P(saved), _native.stream_ptr()))
    torch.cuda.synchronize()
    for buf, n in ((out, m), (hT, bsz), (cT, bsz), (saved, m)):
        assert bool(buf[n:].isnan().all()), 'a row past the end was written'
    return out[:m], hT[:bsz], cT[:bsz], saved[:m]


def backward_kernel(net, dout, saved, c0, bsz, steps, groups=None, envs=None, guard=5):
    """pb_lstm_bptt_backward (groups None) or _rows with the segment view's dPre strides -> (dz, dpre)."""
    hid = net.recurrent.hidden_size
    m, n_act = bsz * steps, net.policy.decoder.weight.shape[0]
    dz, dpre = torch.full((m + guard, 4 * hid), NAN, device='cuda'), torch.full((m + guard, hid), NAN, device='cuda')
    w_cat = net.fused_operands()[4]
    lib = _native.lib()
    if groups is None:
        _native.check(lib.pb_lstm_bptt_backward(
            P(dout), P(saved), P(c0), P(net.gate_weights_transposed()), P(w_cat), bsz, steps, hid, hid, n_act, P(dz),
            P(dpre), _native.stream_ptr()))
    else:
        _native.check(lib.pb_lstm_bptt_backward_rows(
            P(dout), P(saved), P(c0), P(net.gate_weights_transposed()), P(w_cat), bsz, steps, hid, hid, n_act, groups,
            hid, hid * steps * envs, hid * envs, P(dz), P(dpre), _native.stream_ptr()))
    torch.cuda.synchronize()
    assert bool(dz[m:].isnan().all()) and bool(dpre[m:].isnan().all()), 'a row past the end was written'
    return dz[:m], dpre[:m]


def test_envelope_is_refused_outside_128_and_256_before_any_launch():
    """(256, 256) with nothing to do is PB_OK from all five entry points; mismatched sizes, 192 / 384 / 512, 129
    features and 16 actions at H = 256 are PB_ERR_UNSUPPORTED (no device needed: every check comes before any CUDA
    call)."""
    lib = _native.lib()
    p = C.c_void_p(256)

    def sample(size=H, hidden=H, feats=49, n_act=8, m=4):
        return lib.pb_policy_lstm_sample(p, feats, feats, p, p, p, p, p, p, p, 512, p, 512, m, size, hidden, n_act,
                                         C.c_uint64(0), None, None, p, p, p, None, None)

    def fwd(size=H, hidden=H, feats=49, n_act=8, batch=4):
        return lib.pb_lstm_bptt_forward(p, feats, feats, batch, 16, None, None, p, p, p, p, p, p, size, hidden, n_act,
                                        p, p, p, p, None)

    def fwd_rows(size=H, hidden=H, feats=49, n_act=8, batch=4):
        return lib.pb_lstm_bptt_forward_rows(p, feats, batch, 16, 2, 49, 49 * 64, 49 * 4, None, None, p, p, p, p, p, p,
                                             size, hidden, n_act, p, p, p, p, None)

    def bwd(size=H, hidden=H, n_act=8, batch=4):
        return lib.pb_lstm_bptt_backward(p, p, None, p, p, batch, 16, size, hidden, n_act, p, p, None)

    def bwd_rows(size=H, hidden=H, n_act=8, batch=4):
        return lib.pb_lstm_bptt_backward_rows(p, p, None, p, p, batch, 16, size, hidden, n_act, 2, 512, 512 * 64,
                                              512 * 4, p, p, None)
    entries = (sample, fwd, fwd_rows, bwd, bwd_rows)
    assert sample(m=0) == _native.PB_OK
    assert all(f(batch=0) == _native.PB_OK for f in entries[1:])
    for size, hidden in ((256, 128), (128, 256), (192, 192), (384, 384), (512, 512)):
        assert all(f(size=size, hidden=hidden) == _native.PB_ERR_UNSUPPORTED for f in entries), (size, hidden)
    assert all(f(n_act=16) == _native.PB_ERR_UNSUPPORTED for f in entries)
    assert all(f(feats=129) == _native.PB_ERR_UNSUPPORTED for f in (sample, fwd, fwd_rows))


def test_fused_supported_envelope_on_cpu_models():
    """fused_supported accepts H = 128 and 256 with one size everywhere and refuses 192 / 384 / 512, mismatched sizes,
    two layers, 129 features and 16 actions.  The models stay on the CPU; a stand-in carries the observation tensor's
    two attributes the check reads (is_cuda, dtype)."""
    class Cuda:
        is_cuda, dtype = True, torch.float32
    for hidden, ok in ((128, True), (256, True), (192, False), (384, False), (512, False)):
        env = fake_env((49,), 4)
        net = models.LSTMWrapper(env, models.Default(env, hidden_size=hidden), input_size=hidden, hidden_size=hidden)
        assert net.fused_supported(Cuda) == ok, hidden
    env = fake_env((49,), 4)
    mixed = models.LSTMWrapper(env, models.Default(env, hidden_size=256), input_size=256, hidden_size=128)
    two = models.LSTMWrapper(env, models.Default(env, hidden_size=256), input_size=256, hidden_size=256, num_layers=2)
    wide = models.LSTMWrapper(fake_env((129,), 4), models.Default(fake_env((129,), 4), hidden_size=256), 256, 256)
    many = models.LSTMWrapper(fake_env((49,), 16), models.Default(fake_env((49,), 16), hidden_size=256), 256, 256)
    assert not any(n.fused_supported(Cuda) for n in (mixed, two, wide, many))


@gpu
def test_packed_operands_follow_their_layouts():
    """w_gates row 8j + u of chunk ch = gate j of unit 8ch + u of [W_ih | W_hh] (pitch 520, TF32); b_gates in the same
    order; the transposed pack [32][512][40]; w_enc [256][136]."""
    net = make_net(49, 4)
    with torch.no_grad():
        w_enc, b_enc, w_gates, b_gates, w_cat, b_cat = net.fused_operands()
        wt = net.gate_weights_transposed()
    rnn = net.recurrent
    w = rna(torch.cat([rnn.weight_ih_l0, rnn.weight_hh_l0], 1)).float()
    b = rnn.bias_ih_l0 + rnn.bias_hh_l0
    assert tuple(w_enc.shape) == (H, 136) and tuple(w_gates.shape) == (32 * 32, 520) and tuple(wt.shape) == (32 * 512, 40)
    assert tuple(w_cat.shape) == (8, H)
    g3 = w_gates.view(32, 4, 8, 520)
    t3 = wt.view(32, 512, 40)
    for ch in (0, 15, 16, 31):
        for j in range(4):
            rows = H * j + 8 * ch + torch.arange(8, device='cuda')
            assert torch.equal(g3[ch, j, :, :512], w[rows]) and bool((g3[ch, j, :, 512:] == 0).all())
            assert torch.equal(b_gates.view(32, 4, 8)[ch, j], b[rows])
            assert torch.equal(t3[ch, :, 8 * j:8 * j + 8], w[rows].t())
    assert bool((t3[:, :, 32:] == 0).all())


def run_step(pol, x, h0, c0, G=32):
    """One fused step on x with the state as a strided slice of a pool ([m + 2G, 2H] rows, the state in the first H
    columns) and canary rows / columns; -> (a, lp, ent, v, h1, c1, buffers)."""
    m = x.shape[0]
    hbuf = torch.full((m + 2 * G, 2 * H), 7.0, device='cuda')
    cbuf = torch.full((m + 2 * G, 2 * H), 7.0, device='cuda')
    hbuf[G:G + m, :H], cbuf[G:G + m, :H] = h0, c0
    vbuf = torch.full((m + 2 * G,), 7.0, device='cuda')
    lbuf = torch.full((m + 2 * G,), 7.0, device='cuda')
    abuf = torch.full((m + 2 * G,), -7, dtype=torch.int64, device='cuda')
    h, c = hbuf[G:G + m, :H].unsqueeze(0), cbuf[G:G + m, :H].unsqueeze(0)
    with torch.no_grad():
        a, lp, ent, v, (h1, c1) = pol(x, (h, c), out=(vbuf[G:G + m], lbuf[G:G + m], abuf[G:G + m]))
    torch.cuda.synchronize()
    assert h1.data_ptr() == h.data_ptr() and c1.data_ptr() == c.data_ptr()
    return a, ent, (hbuf, cbuf, vbuf, lbuf, abuf)


@gpu
@pytest.mark.parametrize('m', [1, TILE - 1, TILE, TILE + 1, 2 * TILE + 1, 16385])
@pytest.mark.parametrize('n_act', [1, 4, 10, 15])
@pytest.mark.parametrize('feats', [1, 5, 49, 128])
def test_rollout_step_matches_fp64(feats, n_act, m):
    """h', c', value, logprob and entropy vs reference_step within TOL; actions row-exact off the CDF boundaries; the
    counter advances by one; the observations are a column slice with NaN past F and the state a strided pool slice;
    canary rows and columns stay untouched."""
    net = make_net(feats, n_act)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=11).cuda()
    gen = torch.Generator(device='cuda').manual_seed(1000 * feats + m + n_act)
    xw = torch.full((m, feats + 3), NAN, device='cuda')
    xw[:, :feats] = torch.rand(m, feats, device='cuda', generator=gen) * 2 - 1
    x = xw[:, :feats]
    h0 = torch.randn(m, H, device='cuda', generator=gen) * 0.5
    c0 = torch.randn(m, H, device='cuda', generator=gen)
    G = 32
    a, ent, (hbuf, cbuf, vbuf, lbuf, abuf) = run_step(pol, x, h0, c0, G)
    assert int(pol._counter[0]) == 1
    with torch.no_grad():
        h2, c2, out = reference_step(net, x, h0, c0)
    logits, value = out[:, :n_act], out[:, n_act]
    norm = logits - logits.logsumexp(-1, keepdim=True)
    errs = {'h': float((hbuf[G:G + m, :H].double() - h2).abs().max()),
            'c': float((cbuf[G:G + m, :H].double() - c2).abs().max()),
            'value': float((vbuf[G:G + m].double() - value).abs().max()),
            'logprob': float((lbuf[G:G + m].double() - norm.gather(-1, abuf[G:G + m].view(-1, 1)).squeeze(-1)).abs().max()),
            'entropy': float((ent.double() + (norm.exp() * norm).sum(-1)).abs().max())}
    print(f'[lstm256-step] F={feats} n_act={n_act} m={m} max err', {k: f'{e:.2e}' for k, e in errs.items()}, flush=True)
    assert all(e < TOL for e in errs.values()), errs
    assert off_boundary_mismatches(cpu(abuf[G:G + m]), logits, pol._seed, 0) == 0
    for buf, fill in ((hbuf, 7.0), (cbuf, 7.0), (vbuf, 7.0), (lbuf, 7.0), (abuf, -7)):
        assert bool((buf[:G] == fill).all()) and bool((buf[G + m:] == fill).all())
    assert bool((hbuf[:, H:] == 7.0).all()) and bool((cbuf[:, H:] == 7.0).all())


@gpu
def test_rollout_step_rounds_the_upper_half_of_h_prev_to_nearest():
    """Units 128..191 of h_prev hold 1 + 2^-11 (a tie between two TF32 values), units 192..255 hold 1, every other
    operand is zero and W_hh has +1/2 in columns 128..191, -1/2 in 192..255.  cvt.rna rounds the ties up to 1 + 2^-10, so
    every gate pre-activation is 64 * 2^-11 = 2^-5 and h' = 8.0e-3; truncation would give 0 and h' = 0.  The kernel's h'
    matches the rounded-to-nearest restatement within TOL and is farther than 10 * TOL from the truncated one."""
    net = make_net(49, 4)
    rnn = net.recurrent
    with torch.no_grad():
        for p in (rnn.weight_ih_l0, rnn.weight_hh_l0, rnn.bias_ih_l0, rnn.bias_hh_l0):
            p.zero_()
        rnn.weight_hh_l0[:, 128:192] = 0.5
        rnn.weight_hh_l0[:, 192:] = -0.5
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1).cuda()
    m = 130
    x = torch.zeros(m, 49, device='cuda')
    h0 = torch.zeros(m, H, device='cuda')
    h0[:, 128:] = 1.0
    h0[:, 128:192] = 1 + 2 ** -11
    c0 = torch.zeros(m, H, device='cuda')
    _, _, (hbuf, _, _, _, _) = run_step(pol, x, h0, c0)
    got = hbuf[32:32 + m, :H].double()
    with torch.no_grad():
        h_near, _, _ = reference_step(net, x, h0, c0)
        h_trunc, _, _ = reference_step(net, x, torch.where(h0 > 0, torch.ones_like(h0), h0), c0)
    near, trunc = float((got - h_near).abs().max()), float((got - h_trunc).abs().max())
    print(f'[lstm256-tie] vs nearest {near:.2e}, vs truncated {trunc:.2e}', flush=True)
    assert near < TOL and trunc > 10 * TOL, (near, trunc)


@gpu
def test_rollout_step_replays_in_a_cuda_graph():
    """A captured step replayed k times: replay k draws at counter offset k (actions row-exact against the inverse CDF
    of offset k's uniforms), the state is updated in place at every replay."""
    net = make_net(49, 10)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=5).cuda()
    m = 300
    gen = torch.Generator(device='cuda').manual_seed(2)
    x = torch.rand(m, 49, device='cuda', generator=gen)
    h = torch.zeros(1, m, H, device='cuda')
    c = torch.zeros(1, m, H, device='cuda')
    with torch.no_grad():
        pol(x, (h, c))                                   # allocates the counter and the ticket; offset 0
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            a, _, _, _, _ = pol(x, (h, c))
    hr, cr = h[0].double().clone(), c[0].double().clone()
    for k in range(1, 4):
        graph.replay()
        torch.cuda.synchronize()
        with torch.no_grad():
            hr, cr, out = reference_step(net, x, hr, cr)
        assert int(pol._counter[0]) == k + 1
        assert off_boundary_mismatches(cpu(a), out[:, :10], pol._seed, k) == 0, k
        assert float((h[0].double() - hr).abs().max()) < TOL_SEQ


@gpu
@pytest.mark.parametrize('init', [False, True])
@pytest.mark.parametrize('steps', [1, 16])
@pytest.mark.parametrize('bsz', [1, TILE - 1, TILE, TILE + 1, 2 * TILE + 1])
@pytest.mark.parametrize('feats', [1, 49, 128])
def test_forward_matches_fp64(feats, bsz, steps, init):
    """out and (h_T, c_T) vs fp64 (TOL at T = 1, TOL_SEQ at T = 16); no NaN in any output and no row past the end
    written; the saved rows hold h_T, c_T and h0; at T = 1 the value column and (h', c') are bitwise those of the
    rollout step."""
    n_act = 4 if feats != 49 else 15
    net = make_net(feats, n_act)
    gen = torch.Generator(device='cuda').manual_seed(100 * feats + bsz + 7 * steps + int(init))
    x = torch.rand(bsz, steps, feats, device='cuda', generator=gen) * 2 - 1
    h0 = (torch.randn(bsz, H, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(bsz, H, device='cuda', generator=gen) if init else None
    out, hT, cT, saved = forward_kernel(net, x, h0, c0)
    assert all(bool(t.isfinite().all()) for t in (out, hT, cT, saved))
    with torch.no_grad():
        ro, rh, rc = reference_forward(net, x, h0, c0)
    errs = {'out': float((out.double() - ro).abs().max()), 'h': float((hT.double() - rh).abs().max()),
            'c': float((cT.double() - rc).abs().max())}
    print(f'[lstm256-fwd] F={feats} B={bsz} T={steps} init={init} max err', {k: f'{e:.2e}' for k, e in errs.items()},
          flush=True)
    assert all(e < (TOL if steps == 1 else TOL_SEQ) for e in errs.values()), errs
    assert torch.equal(saved[steps - 1::steps, 7 * H:], hT) and torch.equal(saved[steps - 1::steps, 6 * H:7 * H], cT)
    if init:
        assert torch.equal(saved[0::steps, H:2 * H], h0)
    if steps == 1:
        pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1)
        hs = (h0 if init else torch.zeros(bsz, H, device='cuda')).clone().unsqueeze(0)
        cs = (c0 if init else torch.zeros(bsz, H, device='cuda')).clone().unsqueeze(0)
        with torch.no_grad():
            _, _, _, v, (h1, c1) = pol(x[:, 0], (hs, cs))
        torch.cuda.synchronize()
        assert torch.equal(v, out[:, n_act]) and torch.equal(h1[0], hT) and torch.equal(c1[0], cT)


@gpu
@pytest.mark.parametrize('feats,n_act,bsz,steps,init', [
    (49, 4, 37, 16, True), (1, 15, TILE + 1, 16, False), (128, 10, 300, 1, True), (128, 4, 1024, 16, False)])
def test_backward_matches_fp64_autograd(feats, n_act, bsz, steps, init):
    """The ten parameter gradients of forward_packed_seq + backward(dOut) vs fp64 autograd of the same model, each within
    TOL_GRAD of its largest entry (B*T = 16 384 runs the split-K _gemm_tn)."""
    net = make_net(feats, n_act)
    gen = torch.Generator(device='cuda').manual_seed(17 * feats + bsz + steps + n_act)
    x = torch.rand(bsz, steps, feats, device='cuda', generator=gen) * 2 - 1
    keep_relu_off_zero(net, x)
    h0 = (torch.randn(1, bsz, H, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(1, bsz, H, device='cuda', generator=gen) if init else None
    res = net.forward_packed_seq(x, (h0, c0) if init else None)
    assert res is not None
    out, n, (hT, cT) = res
    assert n == n_act and tuple(hT.shape) == (1, bsz, H)
    dout = torch.randn(out.shape, device='cuda', generator=gen) / (bsz * steps) ** 0.5
    dout[:, n_act + 1:] = 0
    net.zero_grad(set_to_none=True)
    out.backward(dout)
    ref = reference_grads_h(net, x, None if h0 is None else h0[0], None if c0 is None else c0[0], dout)
    got = dict(net.policy.named_parameters())
    got.update(dict(net.recurrent.named_parameters()))
    errs = {}
    for name, r in ref.items():
        g = got[name].grad
        assert g is not None and g.shape == r.shape, name
        errs[name] = float((g.double() - r).abs().max()) / (float(r.abs().max()) + 1e-30)
    print(f'[lstm256-bwd] F={feats} n_act={n_act} B={bsz} T={steps} init={init} max err / max |grad|',
          {k: f'{e:.1e}' for k, e in errs.items()}, flush=True)
    assert all(e < TOL_GRAD for e in errs.values()), errs


def reference_grads_h(net, x, h0, c0, dout, pre_grads=None):
    """reference_grads of test_gpu_lstm_bptt.py at the net's hidden size: fp64 autograd with the kernels' operand
    rounding (TF32 leaves for x, W_enc, the gate weights and W_cat; e, h_prev and h' rounded with identity gradient).
    pre_grads: a dict that also receives the gradients pb_lstm_bptt_backward writes, rows b*T + t: 'dz' [B*T, 4H] of the gate
    pre-activations (i, f, g, o) and 'dpre' [B*T, H] of the encoder pre-activation."""
    inner, rnn = net.policy, net.recurrent
    bsz, steps, _ = x.shape
    hid = rnn.hidden_size
    n_act = inner.decoder.weight.shape[0]

    def leaf(t, rounded=True):
        return (rna(t) if rounded else t.detach().double()).clone().requires_grad_(True)
    p = {'encoder.weight': leaf(inner.encoder.weight), 'encoder.bias': leaf(inner.encoder.bias, False),
         'weight_ih_l0': leaf(rnn.weight_ih_l0), 'weight_hh_l0': leaf(rnn.weight_hh_l0),
         'bias_ih_l0': leaf(rnn.bias_ih_l0, False), 'bias_hh_l0': leaf(rnn.bias_hh_l0, False),
         'decoder.weight': leaf(inner.decoder.weight), 'decoder.bias': leaf(inner.decoder.bias, False),
         'value_head.weight': leaf(inner.value_head.weight), 'value_head.bias': leaf(inner.value_head.bias, False)}

    def ste(t):
        return t + (rna(t) - t).detach()
    R = dout.shape[1]
    pad = R - n_act - 1
    w_cat = torch.cat([p['decoder.weight'], p['value_head.weight'], x.new_zeros(pad, hid, dtype=torch.float64)])
    b_cat = torch.cat([p['decoder.bias'], p['value_head.bias'], x.new_zeros(pad, dtype=torch.float64)])
    z0 = torch.zeros(bsz, hid, dtype=torch.float64, device='cuda')
    h = z0 if h0 is None else h0.double()
    c = z0 if c0 is None else c0.double()
    outs, pres, zs = [], [], []
    for t in range(steps):
        pre = rna(x[:, t]) @ p['encoder.weight'].t() + p['encoder.bias']
        e = torch.relu(pre)
        zz = ste(e) @ p['weight_ih_l0'].t() + ste(h) @ p['weight_hh_l0'].t() + p['bias_ih_l0'] + p['bias_hh_l0']
        if pre_grads is not None:
            pre.retain_grad()
            zz.retain_grad()
            pres.append(pre)
            zs.append(zz)
        i, f, g, o = zz.chunk(4, 1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        outs.append(ste(h) @ w_cat.t() + b_cat)
    out = torch.stack(outs, 1).reshape(bsz * steps, R)
    (out * dout.double()).sum().backward()
    if pre_grads is not None:
        pre_grads['dz'] = torch.stack([z.grad for z in zs], 1).reshape(bsz * steps, 4 * hid)
        pre_grads['dpre'] = torch.stack([q.grad for q in pres], 1).reshape(bsz * steps, hid)
    return {k: v.grad for k, v in p.items()}


@gpu
@pytest.mark.parametrize('init', [False, True])
@pytest.mark.parametrize('steps', [1, 16])
@pytest.mark.parametrize('groups', [1, 2, 4])
def test_segment_view_matches_gathered_minibatch(groups, steps, init, fp32_matmul):
    """The _rows entry points on Experience's segment view (E = 150 envs: 150 / 300 / 600 segments leave the last CTA
    ragged) vs the dense ones on the gathered copy: out, h_T, c_T, saved rows and dz bitwise; dPre bitwise after its row
    permutation."""
    feats, n_act, envs = 49, 10, 150
    net = make_net(feats, n_act)
    _, seg, gathered = segment_setup(groups, steps, feats, envs=envs, seed=31 * groups + steps)
    bsz, m = envs * groups, envs * groups * steps
    gen = torch.Generator(device='cuda').manual_seed(7 + groups)
    h0 = (torch.randn(bsz, H, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(bsz, H, device='cuda', generator=gen) if init else None
    ref = forward_kernel(net, gathered, h0, c0)
    got = forward_kernel(net, None, h0, c0, seg=seg)
    for name, a, b in zip(('out', 'h_T', 'c_T', 'saved'), got, ref):
        assert bool(a.isfinite().all()), name
        assert torch.equal(a, b), name
    dout = torch.randn(m, ref[0].shape[1], device='cuda', generator=gen) / m ** 0.5
    dout[:, n_act + 1:] = 0
    dz_ref, dpre_ref = backward_kernel(net, dout, ref[3], c0, bsz, steps)
    dz, dpre = backward_kernel(net, dout, got[3], c0, bsz, steps, groups, envs)
    assert bool(dz.isfinite().all()) and bool(dpre.isfinite().all())
    assert torch.equal(dz, dz_ref)
    assert torch.equal(dpre.view(groups, steps, envs, H).permute(2, 0, 1, 3).reshape(m, H), dpre_ref)


def make_recurrent(env, n, hidden=H, layers=1, seed=3, fused_update=True):
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env, hidden_size=hidden), input_size=hidden,
                             hidden_size=hidden, num_layers=layers)
    sharpen(net)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=seed, fused_update=fused_update).cuda()
    return vec, net, pol


@gpu
@pytest.mark.parametrize('env,n,h,bptt', [('breakout', 256, 32, 16), ('squared', 64, 32, 8)])
def test_train_fused_update_matches_cudnn_update(env, n, h, bptt, monkeypatch):
    """train() at H = 256 with fused_update=True vs False from one snapshot and one rollout, with the bounds of
    test_gpu_lstm_bptt.py::test_train_fused_update_matches_cudnn_update; then the rollout replays bitwise through the
    oracle with the stored actions.  squared's observations (0 / 1 cells, most rows alike) put some of the 256 default-
    initialised encoder units within TF32 rounding of the ReLU kink on many rows at once, and one flipped mask moves a
    whole term of dW_enc between the two paths: its encoder is conditioned with keep_relu_off_zero (|x| <= 1 there)."""
    vec, net, pol = make_recurrent(env, n)
    if env == 'squared':
        keep_relu_off_zero(net, torch.ones(1))
    data = clean_pufferl.create(make_config(n, h, env=env, bptt_horizon=bptt, update_epochs=1), vec, pol)
    clean_pufferl.evaluate(data)
    exp = data.experience
    ora = rollout_oracle(env, n)
    ora.async_reset(1)
    obs_shape = tuple(vec.single_observation_space.shape)
    acts, obs = cpu(exp.actions).reshape(h, n), cpu(exp.obs).reshape(h, n, *obs_shape)
    rew = cpu(exp.rewards).reshape(h, n)
    for t in range(h):
        o, r, _, _, _, _, _ = ora.recv()
        assert np.array_equal(o, obs[t]), t
        assert np.array_equal(np.asarray(r, np.float32).view(np.uint32), rew[t].view(np.uint32)), t
        ora.send(acts[t])
    params0 = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    opt0 = data.optimizer.state_dict()
    res = {}
    for fused in (False, True):
        pol.load_state_dict(params0)
        data.optimizer.load_state_dict(opt0)
        net.invalidate_cache()
        res[fused] = snapshot_train(data, pol, net, fused, monkeypatch)
    (ra, la, pa, path_a), (rb, lb, pb, path_b) = res[True], res[False]
    assert path_a == 'fused' and path_b == 'cudnn', (path_a, path_b)
    gerr = {k: float((ra['grads'][k] - g).abs().max()) / (float(g.abs().max()) + 1e-30) for k, g in rb['grads'].items()}
    serr = [float((a - b).abs().max()) for a, b in zip(ra['states'][1], rb['states'][1])]
    perr = float((pa - pb).abs().max())
    print(f'[lstm256-train] {env} n={n} h={h} bptt={bptt}: grad err / max', {k: f'{e:.1e}' for k, e in gerr.items()},
          f'state err {serr}, param err {perr:.2e}, losses fused {la} cudnn {lb}', flush=True)
    assert set(ra['grads']) == set(rb['grads']) and len(gerr) == 10
    assert all(e < 1.5e-2 for e in gerr.values()), gerr
    assert all(e < 1e-3 for e in serr), serr
    assert np.isclose(la['value_loss'], lb['value_loss'], rtol=3e-2, atol=1e-6), (la['value_loss'], lb['value_loss'])
    assert np.isclose(la['entropy'], lb['entropy'], rtol=1e-4), (la['entropy'], lb['entropy'])
    for k in ('policy_loss', 'approx_kl', 'clipfrac'):
        assert abs(la[k] - lb[k]) < 1e-4, (k, la[k], lb[k])
    assert perr < 2.5e-4, perr
    clean_pufferl.close(data)


@gpu
def test_captured_train_matches_eager_train():
    """train() at H = 256 is captured (train_graph_state == 2, the 'bptt' engine on segment views); a replay agrees with
    an eager train() from the same parameters, Adam state and rollout to 2e-6."""
    env, n, h, bptt = 'breakout', 256, 64, 16
    vec, net, pol = make_recurrent(env, n)
    cfg = make_config(n, h, env=env, bptt_horizon=bptt, update_epochs=2, cuda_graph=True)
    data = clean_pufferl.create(cfg, vec, pol)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
    assert data.train_graph_state == 2, data.msg
    assert data.train_recurrent_path == 'fused' and data.train_minibatch_path == 'segments'
    clean_pufferl.evaluate(data)
    opt = data.optimizer
    params = list(pol.parameters())
    snap_p = [p.detach().clone() for p in params]
    snap_s = [t.clone() for t in adam_state(opt)]
    replays0 = data.train_graph_replays
    clean_pufferl.train(data)
    assert data.train_graph_replays == replays0 + 1
    got = ([p.detach().clone() for p in params], [t.clone() for t in adam_state(opt)], losses(data))
    with torch.no_grad():
        for p, s in zip(params, snap_p):
            p.copy_(s)
        for t, s in zip(adam_state(opt), snap_s):
            t.copy_(s)
    net.invalidate_cache()
    data.config.cuda_graph_train = False
    clean_pufferl.train(data)
    assert data.train_recurrent_path == 'fused'
    ref = ([p.detach() for p in params], adam_state(opt), losses(data))
    perr = max(float((a - b).abs().max()) for a, b in zip(got[0], ref[0]))
    serr = max(float((a.float() - b.float()).abs().max()) for a, b in zip(got[1], ref[1]))
    print(f'[lstm256-graph] param err {perr:.2e}, adam state err {serr:.2e}', flush=True)
    assert perr <= 2e-6 and serr <= 2e-6, (perr, serr)
    clean_pufferl.close(data)


@gpu
@pytest.mark.parametrize('kind', ['hidden384', 'two_layers'])
def test_models_outside_the_envelope_keep_the_unfused_paths(kind):
    """H = 384 and a two-layer H = 256 model: fused_sample=True computes exactly what fused_sample=False computes (the
    kernel never runs) and train() keeps the cuDNN update."""
    hidden, layers = (384, 1) if kind == 'hidden384' else (H, 2)
    n = 64
    vec, net, pol = make_recurrent('squared', n, hidden=hidden, layers=layers)
    x = torch.rand(n, *vec.single_observation_space.shape, device='cuda')
    gen = torch.Generator(device='cuda').manual_seed(9)
    state = (torch.randn(layers, n, hidden, device='cuda', generator=gen),
             torch.randn(layers, n, hidden, device='cuda', generator=gen))
    res = {}
    for fused in (False, True):
        pol.fused_sample = fused
        torch.manual_seed(123)
        with torch.no_grad():
            out = pol(x, (state[0].clone(), state[1].clone()))
        res[fused] = [t.detach().clone() for t in out[:4]] + [s.clone() for s in out[4]]
    assert pol._counter is None
    for u, w in zip(res[False], res[True]):
        assert torch.equal(u, w)
    data = clean_pufferl.create(make_config(n, 16, env='squared', bptt_horizon=8, update_epochs=1), vec, pol)
    clean_pufferl.evaluate(data)
    clean_pufferl.train(data)
    assert data.train_recurrent_path == 'cudnn' and np.isfinite(data.losses.policy_loss)
    clean_pufferl.close(data)


@gpu
def test_memory_learns_with_256_hidden_units():
    """The ocean `memory` env with RecurrentPolicy(LSTMWrapper(Default(hidden_size=256), 256, 256), fused_sample=True,
    fused_update=True): score >= 0.9 within test_gpu_ocean_learning.py's 32-iteration budget, seed 1, on the fused and
    captured update."""
    import test_gpu_ocean_learning as tol
    seed = 1
    torch.manual_seed(seed)
    vec = pvec.make(ocean.env_creator('memory'), num_envs=tol.N, backend=pvec.B200)
    env = vec.driver_env
    net = models.LSTMWrapper(env, models.Default(env, hidden_size=H), input_size=H, hidden_size=H)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=seed, fused_update=True).cuda()
    data = clean_pufferl.create(tol.make_config(seed=seed), vec, pol)
    history, record = [], {}
    for _ in range(tol.BUDGET['memory_lstm']):
        clean_pufferl.evaluate(data)
        history.append(tol.metric('memory_lstm', data))
        if tol.passed('memory_lstm', history[-1]):
            break
        clean_pufferl.train(data)
        record = dict(path=data.train_recurrent_path, form=data.train_minibatch_path, graph=data.train_graph_state)
    clean_pufferl.close(data)
    print(f'[lstm256-memory] iterations {len(history)}, last scores {history[-3:]}, {record}', flush=True)
    assert tol.passed('memory_lstm', history[-1]), (history, record)
    assert record.get('path', 'fused') == 'fused' and record.get('graph', 2) == 2, record
