"""The fused recurrent minibatch update (pb_lstm_bptt_forward / pb_lstm_bptt_backward, csrc/lstm_bptt.cu) behind
models.LSTMWrapper.forward_packed_seq and cleanrl.RecurrentPolicy(fused_update=True).

The forward is checked against an fp64 restatement of its TF32 operand rounding (as test_gpu_policy_lstm.py does for the
rollout step), and at T = 1 against pb_policy_lstm_sample itself; the ten parameter gradients against fp64 autograd of
the same model; train() with fused_update=True against the cuDNN path from one parameter snapshot and one rollout.
Reference: clean_pufferl.py:186-244 (the minibatch update), :188-191 (the [rows, bptt] segments and the state carry)."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from test_gpu_policy_lstm import fake_env, make_config, sharpen
from util_gpu import rna

gpu = pytest.mark.gpu
TOL_STEP = 2e-4         # T = 1 outputs vs fp64 (the rollout step's bound)
TOL_SEQ = 5e-4          # after 16 recurrent steps (the fp64 state is carried, not the kernel's)
TOL_GRAD = 5e-3         # each gradient vs fp64 autograd, relative to that gradient's largest entry (DESIGN.md §4)
P = _native.ptr


def make_net(feats, n_act, hidden=128, layers=1, dtype=np.float32):
    torch.manual_seed(0)
    env = fake_env((feats,), n_act, dtype)
    net = models.LSTMWrapper(env, models.Default(env, hidden_size=hidden), input_size=hidden, hidden_size=hidden,
                             num_layers=layers)
    sharpen(net)
    return net.cuda()


def keep_relu_off_zero(net, x):
    """Encoder pre-activations at least 0.2 away from 0 for every input in [-1, 1]: biases +-0.5 and rows of W_enc with
    L1 norm 0.3.  A TF32-sized change can then not flip a ReLU mask (each flip would move a whole term of dW_enc)."""
    with torch.no_grad():
        w = net.policy.encoder.weight
        w.mul_(0.3 / w.abs().sum(1, keepdim=True))
        b = net.policy.encoder.bias
        b.copy_(0.5 * torch.sign(torch.randn(b.shape, device=b.device, generator=torch.Generator(b.device).manual_seed(3))))
    assert float(x.abs().max()) <= 1.0


def forward_kernel(net, x, h0=None, c0=None, guard=5):
    """pb_lstm_bptt_forward on x [B, T, F] -> (out [B*T, R], h_T, c_T, saved), with NaN canaries past every output."""
    bsz, steps, feats = x.shape
    m = bsz * steps
    n_act = net.policy.decoder.weight.shape[0]
    with torch.no_grad():
        w_enc, b_enc, w_gates, b_gates, w_cat, b_cat = net.fused_operands()
    nan = float('nan')
    out = torch.full((m + guard, w_cat.shape[0]), nan, device='cuda')
    hT, cT = torch.full((bsz + guard, 128), nan, device='cuda'), torch.full((bsz + guard, 128), nan, device='cuda')
    saved = torch.full((m + guard, 1024), nan, device='cuda')
    _native.check(_native.lib().pb_lstm_bptt_forward(
        P(x), x.stride(1), feats, bsz, steps, P(h0), P(c0), P(w_enc), P(b_enc), P(w_gates), P(b_gates), P(w_cat),
        P(b_cat), 128, 128, n_act, P(out), P(hT), P(cT), P(saved), _native.stream_ptr()))
    torch.cuda.synchronize()
    for buf, n in ((out, m), (hT, bsz), (cT, bsz), (saved, m)):
        assert bool(buf[n:].isnan().all()), 'a row past the end was written'
    return out[:m], hT[:bsz], cT[:bsz], saved[:m]


def reference_forward(net, x, h0, c0):
    """fp64 restatement of pb_lstm_bptt_forward (every tensor-core operand rounded to nearest TF32) -> (out [B*T, R],
    h_T, c_T)."""
    inner, rnn = net.policy, net.recurrent
    bsz, steps, _ = x.shape
    w_cat, b_cat = inner.head_matrix()
    h = torch.zeros(bsz, 128, dtype=torch.float64, device='cuda') if h0 is None else h0.double()
    c = torch.zeros(bsz, 128, dtype=torch.float64, device='cuda') if c0 is None else c0.double()
    outs = []
    for t in range(steps):
        e = torch.relu(rna(x[:, t]) @ rna(inner.encoder.weight).t() + inner.encoder.bias.double())
        z = (rna(e) @ rna(rnn.weight_ih_l0).t() + rna(h) @ rna(rnn.weight_hh_l0).t()
             + (rnn.bias_ih_l0 + rnn.bias_hh_l0).double())
        i, f, g, o = z.chunk(4, 1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        outs.append(rna(h) @ rna(w_cat).t() + b_cat.double())
    return torch.stack(outs, 1).reshape(bsz * steps, -1), h, c


def test_unsupported_shapes_are_refused_before_any_launch():
    """PB_ERR_UNSUPPORTED for > 128 features, LSTM sizes other than 128 and more than 15 actions, from both entry points
    (no device needed: the checks come before any CUDA call)."""
    lib = _native.lib()
    p = C.c_void_p(256)

    def fwd(feats=49, size=128, hidden=128, n_act=8, batch=4):
        return lib.pb_lstm_bptt_forward(p, feats, feats, batch, 16, None, None, p, p, p, p, p, p, size, hidden, n_act,
                                        p, p, p, p, None)

    def bwd(size=128, hidden=128, n_act=8, batch=4):
        return lib.pb_lstm_bptt_backward(p, p, None, p, p, batch, 16, size, hidden, n_act, p, p, None)
    assert fwd(feats=129) == _native.PB_ERR_UNSUPPORTED
    assert fwd(size=64) == _native.PB_ERR_UNSUPPORTED
    assert fwd(hidden=256) == _native.PB_ERR_UNSUPPORTED
    assert fwd(n_act=16) == _native.PB_ERR_UNSUPPORTED
    assert bwd(size=64) == _native.PB_ERR_UNSUPPORTED
    assert bwd(hidden=64) == _native.PB_ERR_UNSUPPORTED
    assert bwd(n_act=16) == _native.PB_ERR_UNSUPPORTED
    assert fwd(batch=0) == _native.PB_OK and bwd(batch=0) == _native.PB_OK      # nothing to do


def test_forward_packed_seq_declines_unsupported_models_on_cpu():
    """forward_packed_seq returns None (the caller keeps the cuDNN path) for CPU observations and wrong layouts."""
    torch.manual_seed(0)
    env = fake_env((49,), 4)
    net = models.LSTMWrapper(env, models.Default(env), input_size=128, hidden_size=128)
    assert net.forward_packed_seq(torch.rand(3, 8, 49), None) is None          # not CUDA
    assert net.forward_packed_seq(torch.rand(3, 49), None) is None             # no time axis


@gpu
@pytest.mark.parametrize('init', [False, True])
@pytest.mark.parametrize('steps', [1, 16])
@pytest.mark.parametrize('bsz', [1, 37, 300, 4096])
@pytest.mark.parametrize('n_act', [4, 8, 15])
@pytest.mark.parametrize('feats', [49, 128])
def test_forward_matches_fp64(feats, n_act, bsz, steps, init):
    """out and (h_T, c_T) vs the fp64 restatement; NaN canaries past every output survive; the backward on the same
    segments writes no row past B*T.  At T = 1 the forward is the rollout step: out's value column and (h', c') are
    bitwise those of pb_policy_lstm_sample on the same inputs (both kernels run the cell of lstm_cell.cuh).  Largest errors
    over the 96 cases (H100 80GB HBM3; the kernel is deterministic): T = 1 out 1.4e-4, h 4.2e-5, c 6.6e-5; T = 16
    out 1.8e-4, h 3.9e-5, c 7.0e-5 (out includes the value head, scaled by 3 in sharpen())."""
    net = make_net(feats, n_act)
    gen = torch.Generator(device='cuda').manual_seed(100 * feats + bsz + 7 * steps + n_act + int(init))
    x = torch.rand(bsz, steps, feats, device='cuda', generator=gen) * 2 - 1
    h0 = (torch.randn(bsz, 128, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(bsz, 128, device='cuda', generator=gen) if init else None
    out, hT, cT, saved = forward_kernel(net, x, h0, c0)
    with torch.no_grad():
        ro, rh, rc = reference_forward(net, x, h0, c0)
    errs = {'out': float((out.double() - ro).abs().max()), 'h': float((hT.double() - rh).abs().max()),
            'c': float((cT.double() - rc).abs().max())}
    print(f'[bptt-fwd] F={feats} n_act={n_act} B={bsz} T={steps} init={init} max err',
          {k: f'{e:.2e}' for k, e in errs.items()}, flush=True)
    tol = TOL_STEP if steps == 1 else TOL_SEQ
    assert all(e < tol for e in errs.values()), errs
    # the saved rows hold e, h_prev, the activations, c and h of every step (the backward's inputs)
    assert torch.equal(saved[steps - 1::steps, 896:], hT) and torch.equal(saved[steps - 1::steps, 768:896], cT)
    if init:
        assert torch.equal(saved[0::steps, 128:256], h0)

    # backward over the same segments: dz / dPre rows past B*T untouched
    m, nan = bsz * steps, float('nan')
    dout = torch.randn(m, out.shape[1], device='cuda', generator=gen) * 1e-3
    dz, dpre = torch.full((m + 5, 512), nan, device='cuda'), torch.full((m + 5, 128), nan, device='cuda')
    _, _, _, _, w_cat, _ = net.fused_operands()
    _native.check(_native.lib().pb_lstm_bptt_backward(
        P(dout), P(saved), P(c0), P(net.gate_weights_transposed()), P(w_cat), bsz, steps, 128, 128, n_act, P(dz),
        P(dpre), _native.stream_ptr()))
    torch.cuda.synchronize()
    assert bool(dz[m:].isnan().all()) and bool(dpre[m:].isnan().all())
    assert bool(dz[:m].isfinite().all()) and bool(dpre[:m].isfinite().all())

    if steps == 1:       # the same function as the rollout step
        pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1)
        hs = (h0 if init else torch.zeros(bsz, 128, device='cuda')).clone().unsqueeze(0)
        cs = (c0 if init else torch.zeros(bsz, 128, device='cuda')).clone().unsqueeze(0)
        with torch.no_grad():
            _, _, _, v, (h1, c1) = pol(x[:, 0], (hs, cs))
        torch.cuda.synchronize()
        assert torch.equal(v, out[:, n_act]) and torch.equal(h1[0], hT) and torch.equal(c1[0], cT)


def reference_grads(net, x, h0, c0, dout):
    """fp64 autograd of the model with the kernel's operand rounding: x, W_enc, the gate weights and W_cat enter as their
    TF32 values (leaves), e, h_prev and h' are rounded on the way into each product with an identity gradient."""
    inner, rnn = net.policy, net.recurrent
    bsz, steps, _ = x.shape
    n_act = inner.decoder.weight.shape[0]

    def leaf(t, rounded=True):
        return (rna(t) if rounded else t.detach().double()).clone().requires_grad_(True)
    p = {'encoder.weight': leaf(inner.encoder.weight), 'encoder.bias': leaf(inner.encoder.bias, False),
         'weight_ih_l0': leaf(rnn.weight_ih_l0), 'weight_hh_l0': leaf(rnn.weight_hh_l0),
         'bias_ih_l0': leaf(rnn.bias_ih_l0, False), 'bias_hh_l0': leaf(rnn.bias_hh_l0, False),
         'decoder.weight': leaf(inner.decoder.weight), 'decoder.bias': leaf(inner.decoder.bias, False),
         'value_head.weight': leaf(inner.value_head.weight), 'value_head.bias': leaf(inner.value_head.bias, False)}

    def ste(t):          # rounded value forward, identity backward
        return t + (rna(t) - t).detach()
    R = dout.shape[1]
    pad = R - n_act - 1
    w_cat = torch.cat([p['decoder.weight'], p['value_head.weight'], x.new_zeros(pad, 128, dtype=torch.float64)])
    b_cat = torch.cat([p['decoder.bias'], p['value_head.bias'], x.new_zeros(pad, dtype=torch.float64)])
    h = torch.zeros(bsz, 128, dtype=torch.float64, device='cuda') if h0 is None else h0.double()
    c = torch.zeros(bsz, 128, dtype=torch.float64, device='cuda') if c0 is None else c0.double()
    outs = []
    for t in range(steps):
        e = torch.relu(rna(x[:, t]) @ p['encoder.weight'].t() + p['encoder.bias'])
        z = ste(e) @ p['weight_ih_l0'].t() + ste(h) @ p['weight_hh_l0'].t() + p['bias_ih_l0'] + p['bias_hh_l0']
        i, f, g, o = z.chunk(4, 1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        outs.append(ste(h) @ w_cat.t() + b_cat)
    out = torch.stack(outs, 1).reshape(bsz * steps, R)
    (out * dout.double()).sum().backward()
    return {k: v.grad for k, v in p.items()}


@gpu
@pytest.mark.parametrize('feats,n_act,bsz,steps,init', [
    (49, 4, 37, 16, True), (49, 15, 300, 16, False), (128, 4, 300, 1, True), (128, 8, 37, 16, False),
    (128, 15, 4096, 16, True), (128, 4, 4096, 16, False)])
def test_backward_matches_fp64_autograd(feats, n_act, bsz, steps, init):
    """All ten parameter gradients of forward_packed_seq + backward(dOut) vs fp64 autograd of the same model given the same
    dOut, each within TOL_GRAD of its largest entry.  The encoder pre-activations are kept away from 0
    (keep_relu_off_zero); the zero pad columns of dOut are zero, as pb_ppo_loss writes them.  Largest relative error
    observed over the six cases (H100 80GB HBM3): 8.5e-4 (value_head.weight), all others <= 7.8e-4."""
    net = make_net(feats, n_act)
    gen = torch.Generator(device='cuda').manual_seed(17 * feats + bsz + steps + n_act)
    x = torch.rand(bsz, steps, feats, device='cuda', generator=gen) * 2 - 1
    keep_relu_off_zero(net, x)
    h0 = (torch.randn(1, bsz, 128, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(1, bsz, 128, device='cuda', generator=gen) if init else None
    state = (h0, c0) if init else None
    res = net.forward_packed_seq(x, state)
    assert res is not None
    out, n, (hT, cT) = res
    assert n == n_act and not hT.requires_grad and not cT.requires_grad
    dout = torch.randn(out.shape, device='cuda', generator=gen) / (bsz * steps) ** 0.5
    dout[:, n_act + 1:] = 0
    net.zero_grad(set_to_none=True)
    out.backward(dout)
    ref = reference_grads(net, x, None if h0 is None else h0[0], None if c0 is None else c0[0], dout)
    got = dict(net.policy.named_parameters())
    got.update({k: v for k, v in net.recurrent.named_parameters()})
    errs = {}
    for name, r in ref.items():
        g = got[name].grad
        assert g is not None and g.shape == r.shape, name
        errs[name] = float((g.double() - r).abs().max()) / (float(r.abs().max()) + 1e-30)
    print(f'[bptt-bwd] F={feats} n_act={n_act} B={bsz} T={steps} init={init} max err / max |grad|',
          {k: f'{e:.1e}' for k, e in errs.items()}, flush=True)
    assert all(e < TOL_GRAD for e in errs.values()), errs
    assert got['bias_ih_l0'].grad.data_ptr() != got['bias_hh_l0'].grad.data_ptr()


def snapshot_train(data, pol, net, fused, monkeypatch):
    """One train() with pol.fused_update = fused; -> the first optimizer step's gradients (before clipping), the state
    handed to the second minibatch, the losses and the parameters afterwards."""
    names = {id(p): k for k, p in pol.named_parameters()}
    rec = {'grads': None, 'states': []}
    clip = torch.nn.utils.clip_grad_norm_

    def clip_rec(params, *a, **k):
        params = list(params)
        if rec['grads'] is None:
            rec['grads'] = {names[id(p)]: p.grad.detach().clone() for p in params if p.grad is not None}
        return clip(params, *a, **k)
    monkeypatch.setattr(torch.nn.utils, 'clip_grad_norm_', clip_rec)
    seq, fwd = net.forward_packed_seq, pol.forward

    def seq_rec(x, state=None):
        rec['states'].append(state)
        return seq(x, state)

    def fwd_rec(x, state=None, action=None, out=None):
        rec['states'].append(state)
        return fwd(x, state, action, out)
    monkeypatch.setattr(net, 'forward_packed_seq', seq_rec)
    monkeypatch.setattr(pol, 'forward', fwd_rec)
    pol.fused_update = fused
    clean_pufferl.train(data)
    monkeypatch.undo()
    L = data.losses
    losses = {k: float(getattr(L, k)) for k in ('policy_loss', 'value_loss', 'entropy', 'approx_kl', 'clipfrac')}
    params = torch.cat([p.detach().reshape(-1) for p in pol.parameters()]).clone()
    return rec, losses, params, data.train_recurrent_path


@gpu
@pytest.mark.parametrize('env,n,h,bptt', [('breakout', 256, 32, 16), ('squared', 64, 32, 8)])
def test_train_fused_update_matches_cudnn_update(env, n, h, bptt, monkeypatch):
    """train() with RecurrentPolicy(fused_update=True) vs fused_update=False from one parameter snapshot and one stored
    rollout: the fused path ran; the first minibatch's gradients agree within 1.5e-2 of each parameter's largest entry
    (the DESIGN §4 precedent for two update paths that round at different places); the state handed to the second
    minibatch (the detached final state of the first) agrees; the losses agree; the parameters after one train() are
    within 2.5e-4 (one Adam step is ~lr = 2.5e-4).  Observed (H100 80GB HBM3): breakout gradients within 1.4e-2 (the
    value-head bias; the value head of a freshly initialised policy fits near-zero returns, so its gradient is a nearly
    cancelling mean), state 1.5e-4, parameters 2.5e-5, value loss 2 % apart (7.47e-4 vs 7.62e-4); squared gradients within
    3.4e-4."""
    check_fused_update_matches_cudnn(env, n, h, bptt, monkeypatch)


def check_fused_update_matches_cudnn(env, n, h, bptt, monkeypatch):
    """The body of test_train_fused_update_matches_cudnn_update for env kind `env`, n envs, h steps, bptt horizon bptt."""
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
    sharpen(net)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=3).cuda()
    data = clean_pufferl.create(make_config(n, h, env=env, bptt_horizon=bptt, update_epochs=1), vec, pol)
    clean_pufferl.evaluate(data)
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
    assert len(rb['states']) == len(ra['states']) == 2 and ra['states'][0] is None and rb['states'][0] is None
    serr = [float((a - b).abs().max()) for a, b in zip(ra['states'][1], rb['states'][1])]
    perr = float((pa - pb).abs().max())
    print(f'[bptt-train] {env} n={n} h={h} bptt={bptt}: grad err / max', {k: f'{e:.1e}' for k, e in gerr.items()},
          f'state err {serr}, param err {perr:.2e}, losses fused {la} cudnn {lb}', flush=True)
    assert set(ra['grads']) == set(rb['grads']) and len(gerr) == 10
    assert all(e < 1.5e-2 for e in gerr.values()), gerr
    assert all(e < 1e-3 for e in serr), serr
    # the value loss of a freshly initialised policy differs by ~2 %: a near-zero mean of squared TF32-sized differences
    assert np.isclose(la['value_loss'], lb['value_loss'], rtol=3e-2, atol=1e-6), (la['value_loss'], lb['value_loss'])
    assert np.isclose(la['entropy'], lb['entropy'], rtol=1e-4), (la['entropy'], lb['entropy'])
    for k in ('policy_loss', 'approx_kl', 'clipfrac'):
        assert abs(la[k] - lb[k]) < 1e-4, (k, la[k], lb[k])
    assert perr < 2.5e-4, perr
    clean_pufferl.evaluate(data)
    clean_pufferl.train(data)                  # the fused path again, on the next rollout
    assert data.train_recurrent_path == 'fused' and np.isfinite(data.losses.policy_loss)
    clean_pufferl.close(data)


@gpu
@pytest.mark.parametrize('kind', ['hidden64', 'two_layers', 'uint8_obs', 'fast_path_off'])
def test_unsupported_models_keep_the_cudnn_update(kind, monkeypatch):
    """fused_update=True with a model the kernels do not cover runs the cuDNN path and computes bit-identically what
    fused_update=False computes (same snapshot, same rollout)."""
    env, hidden, layers = ('snake' if kind == 'uint8_obs' else 'squared'), 128, 1
    if kind == 'hidden64':
        hidden = 64
    if kind == 'two_layers':
        layers = 2
    n, h = 64, 16
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env, hidden_size=hidden), input_size=hidden,
                             hidden_size=hidden, num_layers=layers)
    if kind == 'fast_path_off':
        net.policy.fast_path = False
    pol = cleanrl.RecurrentPolicy(net, fused_sample=False, seed=3).cuda()
    data = clean_pufferl.create(make_config(n, h, env=env, bptt_horizon=8, update_epochs=1), vec, pol)
    clean_pufferl.evaluate(data)
    params0 = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    opt0 = data.optimizer.state_dict()
    res = {}
    for fused in (False, True):
        pol.load_state_dict(params0)
        data.optimizer.load_state_dict(opt0)
        net.invalidate_cache()
        res[fused] = snapshot_train(data, pol, net, fused, monkeypatch)
    (ra, la, pa, path_a), (rb, lb, pb, path_b) = res[True], res[False]
    assert path_a == path_b == 'cudnn'
    assert torch.equal(pa, pb) and la == lb
    for k, g in rb['grads'].items():
        assert torch.equal(ra['grads'][k], g), k
    clean_pufferl.close(data)
