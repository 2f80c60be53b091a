"""The recurrent kernels and Default's 8-row update at the shapes the ocean envs give them: 1 to 9 features (memory,
stochastic, multiagent and bandit have 1, password 5 or 7), 1 to 10 actions (2 for most ocean envs, 4 or 10 for bandit),
and row counts at the 128-row CTA edges.

Below 8 features the encoder is a single k-step over an x tile that must be zero past F, W_enc is mostly zero padding,
and the observation rows are not 8-byte aligned; 1 and 2 actions leave most of the 8 head columns as padding, 9 and 10
take the 16-row head instances.  Every check compares with the fp64 restatements of test_gpu_policy_lstm.py and
test_gpu_lstm_bptt.py (TF32 operand rounding modelled), or with the plain modules and autograd, and prints its largest
errors."""
import pytest
import torch

from pufferlib_b200 import models
from test_gpu_default_heads16 import check_fast_path_matches_plain_modules, check_manual_update_matches_autograd
from test_gpu_lstm_bptt import (TOL_GRAD, TOL_SEQ, TOL_STEP, check_fused_update_matches_cudnn, forward_kernel,
                                keep_relu_off_zero, make_net, reference_forward, reference_grads)
from test_gpu_lstm_train_graph import backward_kernel, forward_rows_kernel, segment_setup
from test_gpu_policy_lstm import TOL, check_recurrent_rollout_replays, make_policy, reference_step
from util_gpu import off_boundary_mismatches, rna

pytestmark = pytest.mark.gpu

NAN = float('nan')
PAD = 3                 # observation rows are F + 3 floats apart: a column slice of a wider buffer


def cpu(x):
    return x.detach().cpu().numpy()


def wide_obs(rows, feats, gen):
    """[rows + 2, F + 3] buffer: observations in [-1, 1) in [:rows, :F], NaN in the other columns and the two trailing
    rows.  A kernel that reads a feature past F, or past the last row, gets NaN; its ReLU (fmaxf) turns the NaN
    pre-activations into 0, so the encoder row is wrong, not NaN."""
    wide = torch.full((rows + 2, feats + PAD), NAN, device='cuda')
    wide[:rows, :feats] = torch.rand(rows, feats, device='cuda', generator=gen) * 2 - 1
    return wide


def sliced_obs(rows, feats, gen):
    """Observations [rows, F], rows F + 3 floats apart (wide_obs)."""
    return wide_obs(rows, feats, gen)[:rows, :feats]


# ---- 1. the rollout step, pb_policy_lstm_sample -------------------------------------------------------------------------
FEATS = [1, 5, 7, 8, 9, 127]
ACTS = [1, 2, 7, 9, 10]
ROWS = [1, 127, 128, 129, 257, 16385]
OCEAN = [(1, 2), (5, 2), (7, 2), (1, 4), (1, 10)]           # (F, n_act) of memory / stochastic / multiagent, password,
#                                                            # bandit (4 arms in the goldens, 10 by default)
STEP_CASES = sorted({(f, a, ROWS[(i + j) % len(ROWS)]) for i, f in enumerate(FEATS) for j, a in enumerate(ACTS)}
                    | {(f, a, m) for f, a in OCEAN for m in (129, 16385)})


@pytest.mark.parametrize('feats,n_act,m', STEP_CASES)
def test_rollout_step_matches_fp64(feats, n_act, m):
    """pb_policy_lstm_sample vs the fp64 restatement (reference_step) on every (F, n_act) in FEATS x ACTS, each at one
    row count of ROWS, and on every ocean pair at 129 and 16 385 rows.  Observations are a column
    slice with a row stride of F + 3 and NaN around it, h and c a pool slice with guard rows: h', c', value, logprob and
    entropy within TOL = 2e-4, actions the inverse CDF off a 1e-4 window, guard rows untouched; with one action the
    action is 0 and logprob and entropy are exactly 0.  Largest errors over the 39 cases (H100 80GB HBM3, 700 W power
    limit, one run): value 1.37e-4, c 7.8e-5, h 2.9e-5, logprob 1.3e-5, entropy 8.8e-7."""
    pol = make_policy((feats,), n_act)
    gen = torch.Generator(device='cuda').manual_seed(1000 * feats + m + n_act)
    x = sliced_obs(m, feats, gen)
    assert x.stride(0) == feats + PAD
    h0 = torch.randn(m, 128, device='cuda', generator=gen) * 0.5
    c0 = torch.randn(m, 128, device='cuda', generator=gen)
    G = 32
    hbuf = torch.full((m + 2 * G, 128), 7.0, device='cuda')
    cbuf = torch.full((m + 2 * G, 128), 7.0, device='cuda')
    hbuf[G:G + m], cbuf[G:G + m] = h0, c0
    vbuf = torch.full((m + 2 * G,), 7.0, device='cuda')
    lbuf = torch.full((m + 2 * G,), 7.0, device='cuda')
    abuf = torch.full((m + 2 * G,), -7, dtype=torch.int64, device='cuda')
    h, c = hbuf[G:G + m].unsqueeze(0), cbuf[G:G + m].unsqueeze(0)
    with torch.no_grad():
        a, lp, ent, v, (h1, c1) = pol(x, (h, c), out=(vbuf[G:G + m], lbuf[G:G + m], abuf[G:G + m]))
    torch.cuda.synchronize()
    assert pol._counter is not None and int(pol._counter[0]) == 1          # the kernel ran
    assert h1.data_ptr() == h.data_ptr() and c1.data_ptr() == c.data_ptr()
    with torch.no_grad():
        h2, c2, out = reference_step(pol.policy, x, h0, c0)
    logits, value = out[:, :n_act], out[:, n_act]
    norm = logits - logits.logsumexp(-1, keepdim=True)
    acts = abuf[G:G + m]
    errs = {'h': float((hbuf[G:G + m].double() - h2).abs().max()), 'c': float((cbuf[G:G + m].double() - c2).abs().max()),
            'value': float((vbuf[G:G + m].double() - value).abs().max()),
            'logprob': float((lbuf[G:G + m].double() - norm.gather(-1, acts.view(-1, 1)).squeeze(-1)).abs().max()),
            'entropy': float((ent.double() + (norm.exp() * norm).sum(-1)).abs().max())}
    print(f'[ocean-step] F={feats} n_act={n_act} m={m} max err', {k: f'{e:.2e}' for k, e in errs.items()}, flush=True)
    assert all(e < TOL for e in errs.values()), errs
    assert off_boundary_mismatches(cpu(acts), logits, pol._seed, 0) == 0
    if n_act == 1:
        assert bool((acts == 0).all()) and bool((lbuf[G:G + m] == 0).all()) and bool((ent == 0).all())
    assert int(acts.min()) >= 0 and int(acts.max()) < n_act
    for buf, fill in ((hbuf, 7.0), (cbuf, 7.0), (vbuf, 7.0), (lbuf, 7.0), (abuf, -7)):
        assert bool((buf[:G] == fill).all()) and bool((buf[G + m:] == fill).all())


# ---- 2. the BPTT forward, pb_lstm_bptt_forward --------------------------------------------------------------------------
def sliced_segments(bsz, steps, feats, gen):
    """x [B, T, F] with rows (b, t) F + 3 floats apart (wide_obs).  Sliced after the view, so that stride(1) is the row
    stride at T = 1 too: forward_kernel passes it as the kernel's row stride, and torch gives a size-1 dimension of a
    view of the [B*T, F] slice the stride F."""
    wide = wide_obs(bsz * steps, feats, gen)
    x = wide[:bsz * steps].view(bsz, steps, feats + PAD)[:, :, :feats]
    assert x.stride() == (steps * (feats + PAD), feats + PAD, 1)
    return x


@pytest.mark.parametrize('init', [False, True])
@pytest.mark.parametrize('steps', [1, 16])
@pytest.mark.parametrize('bsz', [127, 128, 129, 257])
@pytest.mark.parametrize('n_act', [1, 2, 10])
@pytest.mark.parametrize('feats', [1, 5, 7, 9])
def test_bptt_forward_matches_fp64(feats, n_act, bsz, steps, init):
    """test_gpu_lstm_bptt.py::test_forward_matches_fp64 at the ocean shapes, around the 128-segment CTA edge, on
    strided observations with NaN around them: out, h_T and c_T vs reference_forward within TOL_STEP (T = 1) / TOL_SEQ
    (T = 16); NaN canaries past every output; at T = 1 the value column and (h', c') bitwise those of
    pb_policy_lstm_sample on the same inputs.  Largest errors over the 192 cases (H100 80GB HBM3, 700 W, one run):
    T = 1 out 9.4e-5, h 1.3e-5, c 3.0e-5; T = 16 out 1.65e-4, h 2.4e-5, c 4.3e-5."""
    net = make_net(feats, n_act)
    gen = torch.Generator(device='cuda').manual_seed(100 * feats + bsz + 7 * steps + n_act + int(init))
    x = sliced_segments(bsz, steps, feats, gen)
    h0 = (torch.randn(bsz, 128, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(bsz, 128, device='cuda', generator=gen) if init else None
    out, hT, cT, _ = forward_kernel(net, x, h0, c0)
    with torch.no_grad():
        ro, rh, rc = reference_forward(net, x, h0, c0)
    errs = {'out': float((out.double() - ro).abs().max()), 'h': float((hT.double() - rh).abs().max()),
            'c': float((cT.double() - rc).abs().max())}
    print(f'[ocean-bptt-fwd] F={feats} n_act={n_act} B={bsz} T={steps} init={init} max err',
          {k: f'{e:.2e}' for k, e in errs.items()}, flush=True)
    tol = TOL_STEP if steps == 1 else TOL_SEQ
    assert all(e < tol for e in errs.values()), errs
    assert bool((out[:, n_act + 1:] == 0).all())            # zero head rows give zero columns
    if steps == 1:
        from pufferlib_b200.frameworks import cleanrl
        pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1)
        hs = (h0 if init else torch.zeros(bsz, 128, device='cuda')).clone().unsqueeze(0)
        cs = (c0 if init else torch.zeros(bsz, 128, device='cuda')).clone().unsqueeze(0)
        with torch.no_grad():
            _, _, _, v, (h1, c1) = pol(x[:, 0], (hs, cs))
        torch.cuda.synchronize()
        assert pol._counter is not None
        assert torch.equal(v, out[:, n_act]) and torch.equal(h1[0], hT) and torch.equal(c1[0], cT)


# ---- 3. the BPTT backward, all ten parameter gradients ------------------------------------------------------------------
def grad_errors(net, ref):
    got = dict(net.policy.named_parameters())
    got.update({k: v for k, v in net.recurrent.named_parameters()})
    errs = {}
    for name, r in ref.items():
        g = got[name].grad
        assert g is not None and g.shape == r.shape, name
        errs[name] = float((g.double() - r).abs().max()) / (float(r.abs().max()) + 1e-30)
    return errs


def encoder_margin(net, x):
    """Smallest |encoder pre-activation| in fp64 on the kernel's operands (TF32 x and W_enc, fp32 bias)."""
    inner = net.policy
    pre = rna(x.reshape(-1, x.shape[-1])) @ rna(inner.encoder.weight).t() + inner.encoder.bias.double()
    return float(pre.abs().min())


BWD_CASES = [(f, a, b) for f, a in [(1, 2), (5, 2), (7, 2), (1, 10), (1, 1)] for b in (129, 257)] + [(1, 2, 1024)]


@pytest.mark.parametrize('feats,n_act,bsz', BWD_CASES)
def test_bptt_backward_matches_fp64_autograd(feats, n_act, bsz):
    """test_gpu_lstm_bptt.py::test_backward_matches_fp64_autograd at the ocean shapes, T = 16, through
    forward_packed_seq on strided observations: the ten parameter gradients vs reference_grads, each within TOL_GRAD of
    its largest entry.  B*T = 16 384 (B = 1024) takes the split-K form of _gemm_tn for the [128, 1] dW_enc, the other
    cases its plain product.  keep_relu_off_zero still keeps every encoder pre-activation at least 0.2 from zero where a row
    of W_enc is one weight (F = 1), up to the TF32 rounding of that weight (2^-11 of 0.3).  Observed over the 11 cases
    (H100 80GB HBM3, 700 W, one run): largest relative error 9.3e-4 (encoder.weight), all others <= 8.1e-4; smallest
    margin 0.2000."""
    steps, init = 16, bsz == 257
    net = make_net(feats, n_act)
    gen = torch.Generator(device='cuda').manual_seed(17 * feats + bsz + steps + n_act)
    x = sliced_segments(bsz, steps, feats, gen)
    keep_relu_off_zero(net, x)
    margin = encoder_margin(net, x)
    assert margin >= 0.1998, margin
    h0 = (torch.randn(1, bsz, 128, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(1, bsz, 128, device='cuda', generator=gen) if init else None
    res = net.forward_packed_seq(x, (h0, c0) if init else None)
    assert res is not None
    out = res[0]
    dout = torch.randn(out.shape, device='cuda', generator=gen) / (bsz * steps) ** 0.5
    dout[:, n_act + 1:] = 0
    net.zero_grad(set_to_none=True)
    out.backward(dout)
    ref = reference_grads(net, x, None if h0 is None else h0[0], None if c0 is None else c0[0], dout)
    errs = grad_errors(net, ref)
    print(f'[ocean-bptt-bwd] F={feats} n_act={n_act} B={bsz} T={steps} init={init} encoder margin {margin:.4f} '
          f'max err / max |grad|', {k: f'{e:.1e}' for k, e in errs.items()}, flush=True)
    assert all(e < TOL_GRAD for e in errs.values()), errs


# ---- 4. segment views vs fp64 -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('init', [False, True])
@pytest.mark.parametrize('groups', [1, 2, 4])
@pytest.mark.parametrize('feats', [1, 5])
def test_segment_view_matches_fp64(feats, groups, init):
    """pb_lstm_bptt_forward_rows / _backward_rows on the segment view of minibatch 1 of 3 (every other row of the
    rollout buffer NaN; 150 envs, T = 16, 2 actions) vs fp64, not only vs the dense kernel: out, h_T and c_T vs
    reference_forward on the gathered copy within TOL_SEQ; dW_enc from the slab form of _gemm_tn on the kernel's dPre
    vs the encoder.weight gradient of reference_grads within TOL_GRAD of its largest entry.  Largest errors over the
    12 cases (H100 80GB HBM3, 700 W, one run): out 1.3e-4, h 2.0e-5, c 3.9e-5, dW_enc 8.6e-4 of its largest entry."""
    steps, n_act, envs = 16, 2, 150
    net = make_net(feats, n_act)
    _, seg, gathered = segment_setup(groups, steps, feats, envs=envs, seed=31 * groups + feats + int(init))
    keep_relu_off_zero(net, gathered)
    bsz, m = envs * groups, envs * groups * steps
    gen = torch.Generator(device='cuda').manual_seed(7 + feats + groups)
    h0 = (torch.randn(bsz, 128, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(bsz, 128, device='cuda', generator=gen) if init else None
    out, hT, cT, saved = forward_rows_kernel(net, seg, h0, c0)
    with torch.no_grad():
        ro, rh, rc = reference_forward(net, gathered, h0, c0)
    errs = {'out': float((out.double() - ro).abs().max()), 'h': float((hT.double() - rh).abs().max()),
            'c': float((cT.double() - rc).abs().max())}
    dout = torch.randn(m, out.shape[1], device='cuda', generator=gen) / m ** 0.5
    dout[:, n_act + 1:] = 0
    _, dpre = backward_kernel(net, dout, saved, c0, bsz, steps, groups, envs)
    slabs = seg.permute(1, 2, 0, 3).view(groups, steps * envs, feats)
    dw_enc = models._gemm_tn(dpre, slabs)
    ref = reference_grads(net, gathered, h0, c0, dout)['encoder.weight']
    errs['dW_enc'] = float((dw_enc.double() - ref).abs().max()) / (float(ref.abs().max()) + 1e-30)
    print(f'[ocean-segments] F={feats} G={groups} init={init} max err', {k: f'{e:.2e}' for k, e in errs.items()},
          flush=True)
    assert errs['out'] < TOL_SEQ and errs['h'] < TOL_SEQ and errs['c'] < TOL_SEQ, errs
    assert errs['dW_enc'] < TOL_GRAD, errs


# ---- 5. train() and evaluate() on the ocean envs ------------------------------------------------------------------------
@pytest.mark.parametrize('env', ['memory', 'password', 'bandit'])
def test_train_fused_update_matches_cudnn_update_on_ocean_envs(env, monkeypatch):
    """test_gpu_lstm_bptt.py::test_train_fused_update_matches_cudnn_update on memory (F = 1, 2 actions), password
    (F = 5, 2 actions) and the 10-arm bandit (F = 1): 128 envs x 32 steps, bptt 16, same tolerances.  Observed (H100
    80GB HBM3, 700 W, one run): gradients within 9.3e-4 of their largest entry (bandit weight_ih_l0; memory 3.7e-4,
    password 3.3e-4), state 2.0e-4, parameters 2.0e-5, value loss 4.5e-5 relative, the other losses 2.3e-7 apart."""
    check_fused_update_matches_cudnn(env, 128, 32, 16, monkeypatch)


@pytest.mark.parametrize('env', ['memory', 'password'])
def test_fused_recurrent_rollout_replays_on_ocean_envs(env):
    """test_gpu_policy_lstm.py::test_fused_recurrent_rollout_replays on memory and password, 128 envs x 64 steps,
    replayed through oracle.ocean.OceanSerial: env rows bitwise, values / logprobs / final lstm_h / lstm_c within
    TOL_ROLLOUT of the fp64 recurrence, draws off-boundary exact.  Observed (H100 80GB HBM3, 700 W, one run): value
    1.26e-4, logprob 1.3e-5, lstm_h 1.4e-5, lstm_c 2.7e-5."""
    check_recurrent_rollout_replays(env, 128, 64)


# ---- 6. Default on 8-row heads at small F -------------------------------------------------------------------------------
@pytest.mark.parametrize('n_act', [1, 2, 7])
@pytest.mark.parametrize('features', [1, 5, 7])
def test_default_8_row_fast_path_matches_plain_modules(features, n_act):
    """test_gpu_default_heads16.py::test_default_16_row_fast_path_matches_plain_modules on [M, 8] heads at 1, 5 and 7
    features, M = 1, 37, 4096, 70001, same tolerances (outputs 2e-3, gradients 5e-3 of their largest entry).
    Observed (H100 80GB HBM3, 700 W, one run): outputs bitwise equal, gradients within 1.06e-3 of their largest entry
    (F = 1, 2 actions)."""
    check_fast_path_matches_plain_modules(features, n_act)


@pytest.mark.parametrize('env', ['memory', 'password', 'stochastic'])
def test_manual_update_8_rows_matches_autograd_update(env):
    """test_gpu_default_heads16.py::test_manual_update_16_rows_matches_autograd_update with head_rows == 8 on memory,
    password and stochastic (2 actions): the hand-written chain on slabs vs autograd + clip_grad_norm_ +
    torch.optim.Adam, parameters within 2e-5, losses within 1e-4.  Observed (H100 80GB HBM3, 700 W, one run):
    parameters 6.0e-8 apart, losses 9.0e-6 relative."""
    check_manual_update_matches_autograd(env, 2)
