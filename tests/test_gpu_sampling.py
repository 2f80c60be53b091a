"""The action samplers held row by row to a plain restatement: pb_sample_logits (csrc/sample.cu), pb_policy_mlp_sample
(csrc/policy_mlp.cu) and, under a shifted head bias, pb_policy_lstm_sample.  All of them draw with pb_sample_row
(csrc/policy_sample.cuh): the first k with u' < c_k, the running sums of p_k = exp(z_k - lse), where u' = u, or u times
their total T when a large common offset has left T more than 2^-20 from 1.

The restatement draws from fp64 probabilities with the same counter-based uniforms (util_gpu.uniforms); a row's action
must match unless its u lies within a small window of a CDF boundary, where the kernel's fp32 weights may decide either
way.  Kernel inputs are exact fp32 values, and where the kernel rounds tensor-core operands to TF32 the restatement
does too (cvt.rna: util_gpu.rna), so the logprob / entropy / value bounds are tight.  Reference:
frameworks/cleanrl.py:25-47 (sample_logits), :12-23 (entropy)."""
import ctypes as C

import numpy as np
import pytest
import torch

from pufferlib_b200 import _native, models
from pufferlib_b200.frameworks import cleanrl
from test_gpu_policy_lstm import fake_env, make_policy, reference_step
from util_gpu import restated_draw, rna, softmax64, uniforms

gpu = pytest.mark.gpu
DEV = 'cuda'
P = _native.ptr
G = 32                    # canary rows after each output
TOL = 1e-5                # pb_sample_logits: logprob / entropy vs fp64 of the same fp32 logits
TOL_MLP = 2e-4            # pb_policy_mlp_sample outputs vs the fp64 restatement of its TF32 rounding
WIN = 1e-5                # boundary window for exact logits
WIN_MLP = 1e-4            # boundary window for restated (TF32) logits
OUTPUTS = ('actions', 'logprobs', 'entropies', 'values_row', 'logprobs_row', 'actions_row')


def cpu(x):
    return x.detach().cpu().numpy()


def out_buffers(n):
    """The six outputs of pb_sample_logits, n rows + G canary rows each."""
    return {k: (torch.full((n + G,), -7, dtype=torch.int64, device=DEV) if k.startswith('actions')
                else torch.full((n + G,), 7.0, device=DEV)) for k in OUTPUTS}


def sample_logits(logits, n, n_act, seed, offset, offset_dev=None, value=None, vstride=0, bufs=None, null=()):
    """pb_sample_logits on torch views; outputs named in `null` are passed as NULL."""
    b = {k: (None if k in null or (k == 'values_row' and value is None) else v) for k, v in bufs.items()}
    _native.check(_native.lib().pb_sample_logits(
        P(logits), logits.stride(0), n, n_act, C.c_uint64(seed), C.c_uint64(offset), P(offset_dev), P(b['actions']),
        P(b['logprobs']), P(b['entropies']), P(value), vstride, P(b['values_row']), P(b['logprobs_row']),
        P(b['actions_row']), _native.stream_ptr()))
    torch.cuda.synchronize()


def fp64_logprob_entropy(logits, actions):
    """fp64 normalized[a] and -sum(p * normalized) of the fp32 logits (torch, any device)."""
    z = logits.double()
    norm = z - z.logsumexp(-1, keepdim=True)
    p = norm.exp()
    ent = -(p * norm.clamp(min=-1e300)).sum(-1)
    return norm.gather(-1, actions.view(-1, 1)).squeeze(-1), ent


# ---------------------------------------------------------------------------------------------------------------------
# C ABI refusals (no device needed: the checks come before any CUDA call)

def test_sample_logits_refusals():
    lib, p = _native.lib(), C.c_void_p(256)

    def call(n_act=4, stride=4, value=p, values_row=None):
        return lib.pb_sample_logits(p, stride, 10, n_act, C.c_uint64(0), C.c_uint64(0), None, p, p, p, value, 8,
                                    values_row, None, None, None)
    assert call(n_act=0, stride=8) == _native.PB_ERR_UNSUPPORTED
    assert call(n_act=33, stride=40) == _native.PB_ERR_UNSUPPORTED
    assert call(n_act=8, stride=7) == _native.PB_ERR_INVALID
    assert call(value=None, values_row=p) == _native.PB_ERR_INVALID


# ---------------------------------------------------------------------------------------------------------------------
# pb_sample_logits row by row

@gpu
@pytest.mark.parametrize('n', [1, 255, 257, 100003])
@pytest.mark.parametrize('n_act', [1, 2, 4, 7, 8, 15, 16, 18, 31, 32])
def test_sample_logits_row_exact(n_act, n):
    """Logits as a column slice of wider rows (stride n_act + 3) and, for n_act <= 15, as the packed 8 / 16 head rows
    of cleanrl.Policy._sample_fused (value in column n_act, value stride 8 or 16).  The uniform is drawn at
    offset + *offset_dev = 3 + 2^40 + 7.  Every action is the restated inverse CDF off the 1e-5 boundary windows;
    logprob and entropy are within 1e-5 of fp64; values_row / logprobs_row / actions_row copy value / logprob / action;
    each output in turn may be NULL without changing the others; nothing is written past row n."""
    gen = torch.Generator(device=DEV).manual_seed(1000 * n_act + n)
    seed, offset, dev_off = 11 + n_act, 3, 2 ** 40 + 7
    offset_dev = torch.tensor([dev_off], dtype=torch.int64, device=DEV)
    u = uniforms(seed, offset + dev_off, n)
    layouts = ['slice'] + (['packed'] if n_act <= 15 else [])
    for layout in layouts:
        if layout == 'slice':
            wide = torch.randn(n, n_act + 3, device=DEV, generator=gen) * 3
            logits = wide[:, :n_act]
            vs = 8 if n_act % 2 else 16
            vsrc = torch.randn(n, vs, device=DEV, generator=gen)
            value = vsrc[:, 5]
        else:
            vs = 8 if n_act + 1 <= 8 else 16
            packed = torch.randn(n, vs, device=DEV, generator=gen) * 3
            packed[:, n_act + 1:] = 0
            logits, value = packed[:, :n_act], packed[:, n_act]
        assert logits.stride(0) in (n_act + 3, vs) and value.stride(0) == vs
        full = out_buffers(n)
        sample_logits(logits, n, n_act, seed, offset, offset_dev, value, vs, full)
        acts = full['actions'][:n]
        assert int(acts.min()) >= 0 and int(acts.max()) < n_act
        want, near = restated_draw(softmax64(logits), u, WIN)
        bad = int(((want != cpu(acts)) & ~near).sum())
        assert bad == 0, (layout, bad, int(near.sum()))
        lp64, ent64 = fp64_logprob_entropy(logits, acts)
        e_lp = float((full['logprobs'][:n].double() - lp64).abs().max())
        e_ent = float((full['entropies'][:n].double() - ent64).abs().max())
        assert e_lp < TOL and e_ent < TOL, (layout, e_lp, e_ent)
        assert torch.equal(full['actions_row'][:n], acts) and torch.equal(full['logprobs_row'][:n], full['logprobs'][:n])
        assert torch.equal(full['values_row'][:n], value)
        for k, buf in full.items():
            assert bool((buf[n:] == (-7 if k.startswith('actions') else 7.0)).all()), (layout, k)
        for drop in OUTPUTS:
            part = out_buffers(n)
            sample_logits(logits, n, n_act, seed, offset, offset_dev, value, vs, part, null=(drop,))
            for k, buf in part.items():
                if k == drop:
                    assert bool((buf == (-7 if k.startswith('actions') else 7.0)).all()), (layout, drop)
                else:
                    assert torch.equal(buf, full[k]), (layout, drop, k)


@gpu
@pytest.mark.parametrize('shift', [0.0, 1e3, 1e5, 1e7])
def test_sample_logits_shift_invariance(shift):
    """softmax is shift-invariant and so is the draw: fixed rows [0, 0] and [0, -1.5] and random 4- and 16-action rows,
    each plus a common offset C.  The logits are the fp32 values base + C and the restatement starts from those same
    fp32 values.  Actions are row-exact off the 1e-5 windows.  Logprob is within max(1e-5, ulp(C)) of
    cleanrl.sample_logits on the same actions, entropy within 1e-5 of cleanrl.entropy where torch's fp32 logsumexp
    rounds like the kernel's (lse = z_a - logprob, exact here) and within their difference + 1e-5 elsewhere.
    A draw from a CDF built as exp(z - lse) misses 1 by up to ulp(C) / 2 and fails here from C = 1e5 on."""
    ulp = float(np.spacing(np.float32(shift))) if shift else 0.0
    gen = torch.Generator(device=DEV).manual_seed(7)
    n = 1 << 16
    cases = {'[0, 0]': torch.zeros(n, 2, device=DEV),
             '[0, -1.5]': torch.tensor([0.0, -1.5], device=DEV).repeat(n, 1),
             'random 4': torch.randn(n, 4, device=DEV, generator=gen) * 2,
             'random 16': torch.randn(n, 16, device=DEV, generator=gen) * 2}
    for ci, (name, base) in enumerate(cases.items()):
        logits = (base.double() + shift).float().contiguous()
        n_act = logits.shape[1]
        seed = 100 + ci
        bufs = out_buffers(n)
        sample_logits(logits, n, n_act, seed, 0, bufs=bufs)
        acts = bufs['actions'][:n]
        want, near = restated_draw(softmax64(logits), uniforms(seed, 0, n), WIN)
        bad = int(((want != cpu(acts)) & ~near).sum())
        freq = np.bincount(cpu(acts), minlength=n_act)[:2] / n
        print(f'[shift {shift:g}] {name}: {bad} rows off the restated draw, first frequencies {freq}', flush=True)
        assert bad == 0, (name, bad)
        _, ref_lp, _ = cleanrl.sample_logits(logits, acts)
        lp = bufs['logprobs'][:n]
        e_lp = float((lp - ref_lp).abs().max())
        assert e_lp <= max(TOL, ulp), (name, e_lp)
        ref_lse = logits.logsumexp(-1).double()
        k_lse = logits.gather(-1, acts.view(-1, 1)).squeeze(-1).double() - lp.double()
        ref_ent = cleanrl.entropy(logits - logits.logsumexp(-1, keepdim=True))
        d_ent = (bufs['entropies'][:n].double() - ref_ent.double()).abs()
        differ = (k_lse != ref_lse) if shift >= 1e3 else torch.zeros_like(d_ent, dtype=torch.bool)
        if int(differ.sum()):
            print(f'[shift {shift:g}] {name}: {int(differ.sum())} rows where torch logsumexp rounds unlike the kernel',
                  flush=True)
        bound = torch.where(differ, (k_lse - ref_lse).abs() + TOL, torch.full_like(d_ent, TOL))
        assert bool((d_ent <= bound).all()), (name, float(d_ent.max()))


@gpu
def test_sample_logits_impossible_actions():
    """2^24 rows with zero-weight actions: -inf logits and logits more than 104 below the row's maximum (exp gives 0 in
    fp32), placed last, interleaved and first.  No row draws one.  Rows with u >= 1 - 2^-20 are checked one by one
    against the restatement; (seed 1, offset 5) puts u = 0 exactly on row 14 212 428, whose action 0 has zero weight
    and must not be drawn.  With n_act = 1 the action is 0 and logprob and entropy are 0."""
    n, n_act, seed, offset, zero_row = 1 << 24, 6, 1, 5, 14212428
    u = uniforms(seed, offset, n)
    assert u[zero_row] == 0.0
    gen = torch.Generator(device=DEV).manual_seed(3)
    logits = torch.randn(n, n_act, device=DEV, generator=gen)
    kind = torch.arange(n, device=DEV) % 3
    impossible = torch.zeros(n, n_act, dtype=torch.bool, device=DEV)
    impossible[kind == 0, 4:] = True                       # last
    impossible[kind == 1, 0::2] = True                     # interleaved
    impossible[kind == 2, 0] = impossible[kind == 2, 3] = True     # first and inside
    impossible[zero_row] = False
    impossible[zero_row, 0] = True
    mx = logits.masked_fill(impossible, -float('inf')).max(-1, keepdim=True).values
    far = torch.arange(n_act, device=DEV).view(1, -1) % 2 == 1        # odd columns: finite, 104.5 .. 120 below the max
    low = mx - 104.5 - 15 * torch.rand(n, n_act, device=DEV, generator=gen)
    logits = torch.where(impossible, torch.where(far, low, torch.full_like(low, -float('inf'))), logits)
    logits[zero_row, 0] = -float('inf')
    assert bool((torch.exp(logits[impossible] - mx.expand(-1, n_act)[impossible]) == 0).all())
    bufs = {k: torch.empty(n, dtype=torch.int64 if k == 'actions' else torch.float32, device=DEV)
            for k in ('actions', 'logprobs', 'entropies')}
    bufs.update(values_row=None, logprobs_row=None, actions_row=None)
    _native.check(_native.lib().pb_sample_logits(
        P(logits), n_act, n, n_act, C.c_uint64(seed), C.c_uint64(offset), None, P(bufs['actions']), P(bufs['logprobs']),
        P(bufs['entropies']), None, 0, None, None, None, _native.stream_ptr()))
    torch.cuda.synchronize()
    acts = bufs['actions']
    drawn_impossible = int(impossible.gather(-1, acts.view(-1, 1)).sum())
    assert drawn_impossible == 0, drawn_impossible
    assert int(acts[zero_row]) == 1
    probs = torch.softmax(logits.double(), -1)
    cdf = probs.cumsum(-1)
    ut = torch.from_numpy(u.astype(np.float64)).to(DEV)
    want = (ut[:, None] >= cdf).sum(-1).clamp(max=n_act - 1)
    near = ((ut[:, None] - cdf[:, :-1]).abs() < WIN).any(-1)
    bad = int(((want != acts) & ~near).sum())
    assert bad == 0, bad
    top = np.flatnonzero(u >= 1 - 2.0 ** -20)
    print(f'[impossible] {len(top)} rows with u >= 1 - 2^-20; near-boundary rows {int(near.sum())}', flush=True)
    assert len(top) > 0
    for r in top:
        row = logits[r].tolist()
        print(f'  row {r}: u = 1 - {1 - float(u[r]):.3e}, logits {[f"{x:.3g}" for x in row]}, action {int(acts[r])}, '
              f'restated {int(want[r])}', flush=True)
        assert int(acts[r]) == int(want[r]) and not bool(impossible[r, int(acts[r])]), r
    # the logprob of a drawn action is finite and the entropy matches fp64 (the -inf terms contribute 0)
    lp64, ent64 = fp64_logprob_entropy(logits, acts)
    assert float((bufs['logprobs'].double() - lp64).abs().max()) < TOL
    assert float((bufs['entropies'].double() - ent64).abs().max()) < TOL
    # a single action
    one = torch.cat([torch.randn(250, 1, device=DEV, generator=gen) * 10, torch.tensor(
        [[0.0], [1e7], [-1e7], [3e38], [-3e38], [1e-30], [-104.5]], device=DEV)])
    b1 = out_buffers(one.shape[0])
    sample_logits(one, one.shape[0], 1, seed, offset, bufs=b1)
    m = one.shape[0]
    assert bool((b1['actions'][:m] == 0).all()) and bool((b1['logprobs'][:m] == 0).all())
    assert bool((b1['entropies'][:m] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# pb_policy_mlp_sample against fp64

def make_default(n_act, seed=0, feats=128):
    torch.manual_seed(seed)
    net = models.Default(fake_env((feats,), n_act)).to(DEV)
    with torch.no_grad():            # informative heads: the 0.01-std init gives near-uniform policies
        net.decoder.weight.mul_(20.0)
        net.decoder.bias.uniform_(-1, 1)
    net.invalidate_cache()
    return net


def mlp_reference(x, w_enc, b_enc, w_cat, b_cat):
    """fp64 restatement of pb_policy_mlp_sample's head outputs -> (head product [m, R], head product + bias)."""
    h = torch.relu(rna(x) @ rna(w_enc).t() + b_enc.double())
    prod = rna(h) @ rna(w_cat).t()
    return prod, prod + b_cat.double()


def check_mlp_outputs(out64, n_act, acts, lp, ent, val, seed, offset, tag):
    logits, value = out64[:, :n_act], out64[:, n_act]
    lp64, ent64 = fp64_logprob_entropy(logits, acts)
    errs = {'value': float((val.double() - value).abs().max()), 'logprob': float((lp.double() - lp64).abs().max())}
    if ent is not None:
        errs['entropy'] = float((ent.double() - ent64).abs().max())
    want, near = restated_draw(softmax64(logits), uniforms(seed, offset, acts.shape[0]), WIN_MLP)
    bad = int(((want != cpu(acts)) & ~near).sum())
    print(f'[policy-mlp] {tag} max err', {k: f'{e:.2e}' for k, e in errs.items()}, f'near-boundary rows {int(near.sum())}',
          flush=True)
    assert all(e < TOL_MLP for e in errs.values()), errs
    assert bad == 0, bad
    return errs


MLP_CASES = [(20001, a) for a in range(1, 16)] + [(m, a) for a in (1, 7, 8, 15) for m in (1, 63, 64, 65, 16384)]


@gpu
@pytest.mark.parametrize('m,n_act', MLP_CASES)
def test_policy_mlp_kernel_matches_fp64(m, n_act):
    """cleanrl.Policy's one-kernel step vs rna(x) @ rna(W_enc)^T + b -> relu -> rna(h) @ rna(W_cat)^T + b_cat in fp64:
    value, logprob and entropy within 2e-4, actions row-exact off the 1e-4 windows, guard rows around the output rows
    untouched, the counter advanced by one and the exit ticket back at 0."""
    net = make_default(n_act, seed=m + n_act)
    pol = cleanrl.Policy(net, fused_sample=True, seed=9 + n_act)
    gen = torch.Generator(device=DEV).manual_seed(m * 31 + n_act)
    x = torch.rand(m, 128, device=DEV, generator=gen) * 2 - 1
    vbuf, lbuf = torch.full((m + 2 * G,), 7.0, device=DEV), torch.full((m + 2 * G,), 7.0, device=DEV)
    abuf = torch.full((m + 2 * G,), -7, dtype=torch.int64, device=DEV)
    with torch.no_grad():
        a, lp, ent, v = pol(x, out=(vbuf[G:G + m], lbuf[G:G + m], abuf[G:G + m]))
        w_cat, b_cat = net.head_matrix()
        _, out64 = mlp_reference(x, net.encoder.weight, net.encoder.bias, w_cat, b_cat)
    torch.cuda.synchronize()
    assert pol._ticket is not None and a.data_ptr() == abuf[G:].data_ptr()
    check_mlp_outputs(out64, n_act, abuf[G:G + m], lbuf[G:G + m], ent, vbuf[G:G + m], pol._seed, 0,
                      f'm={m} n_act={n_act}')
    for buf, fill in ((vbuf, 7.0), (lbuf, 7.0), (abuf, -7)):
        assert bool((buf[:G] == fill).all()) and bool((buf[G + m:] == fill).all())
    assert int(pol._counter[0]) == 1 and int(pol._ticket[0]) == 0


@gpu
@pytest.mark.parametrize('n_act', [3, 12])
def test_policy_mlp_kernel_through_the_abi(n_act):
    """pb_policy_mlp_sample called directly: observation rows 132 floats apart inside a larger buffer, entropies NULL,
    the counter preset to 2^33 + 5 (the draw uses that offset; afterwards it is 2^33 + 6 and the ticket 0)."""
    m, start = 1000, 2 ** 33 + 5
    net = make_default(n_act, seed=77)
    gen = torch.Generator(device=DEV).manual_seed(5)
    buf = torch.full((m + 3, 132), 9.0, device=DEV)
    buf[1:m + 1, :128] = torch.rand(m, 128, device=DEV, generator=gen) * 2 - 1
    x = buf[1:m + 1, :128]
    counter = torch.tensor([start], dtype=torch.int64, device=DEV)
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    acts = torch.full((m,), -7, dtype=torch.int64, device=DEV)
    lp, val = torch.full((m,), 7.0, device=DEV), torch.full((m,), 7.0, device=DEV)
    w_enc = models._round_tf32(net.encoder.weight)
    w_cat, b_cat = net.head_matrix(cache=False)
    _native.check(_native.lib().pb_policy_mlp_sample(
        P(x), 132, P(w_enc), P(net.encoder.bias), P(w_cat), P(b_cat), m, 128, 128, n_act, C.c_uint64(4), P(counter),
        P(ticket), P(acts), P(lp), P(val), None, _native.stream_ptr()))
    torch.cuda.synchronize()
    with torch.no_grad():
        _, out64 = mlp_reference(x, net.encoder.weight, net.encoder.bias, w_cat, b_cat)
    check_mlp_outputs(out64, n_act, acts, lp, None, val, 4, start, f'abi n_act={n_act}')
    assert int(counter[0]) == start + 1 and int(ticket[0]) == 0


TIE = 1.0 + 2.0 ** -11      # halfway between two TF32 values: cvt.rna, round-to-nearest-even and truncation all differ


@gpu
@pytest.mark.parametrize('n_act', [3, 10])
@pytest.mark.parametrize('probe', ['x', 'relu_h', 'head_row', 'w_enc_policy'])
def test_policy_mlp_tf32_rounding_probes(probe, n_act):
    """Inputs on an exact TF32 tie 1 + 2^-11, so that the value moves by >= 4.8e-4 (more than the 2e-4 bound) if an
    operand is rounded any other way than cvt.rna: x with W_enc = I; x = 0 with b_enc at the tie (the rounding of
    relu(h)); the value row of the head matrix at the tie; W_enc at the tie passed through cleanrl.Policy (the rounding
    of models.Default.encoder_weight_tf32).  Row j probes hidden unit j; n_act 3 and 10 take the 8- and 16-row heads."""
    m = 128
    torch.manual_seed(n_act)
    net = models.Default(fake_env((128,), n_act)).to(DEV)
    eye = torch.eye(128, device=DEV)
    with torch.no_grad():
        net.encoder.weight.copy_(eye * (TIE if probe == 'w_enc_policy' else 1.0))
        net.encoder.bias.fill_(TIE if probe == 'relu_h' else 0.0)
        net.decoder.weight.normal_(0, 0.5)
        net.decoder.bias.uniform_(-1, 1)
        net.value_head.weight.fill_(TIE if probe == 'head_row' else 1.0)
        net.value_head.bias.zero_()
    net.invalidate_cache()
    x = torch.zeros(m, 128, device=DEV) if probe == 'relu_h' else eye * (TIE if probe == 'x' else 1.0)
    pol = cleanrl.Policy(net, fused_sample=True, seed=3)
    with torch.no_grad():
        a, lp, ent, v = pol(x)
        w_cat, b_cat = net.head_matrix()
        _, out64 = mlp_reference(x, net.encoder.weight, net.encoder.bias, w_cat, b_cat)
    torch.cuda.synchronize()
    value = out64[:, n_act]
    trunc = lambda t: (t.detach().float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32).double()  # noqa
    h_t = torch.relu(trunc(x) @ trunc(net.encoder.weight).t() + net.encoder.bias.double())
    v_trunc = (trunc(h_t) @ trunc(w_cat).t() + b_cat.double())[:, n_act]
    assert float((value - v_trunc).abs().min()) >= 4.8e-4             # the probe separates the roundings
    check_mlp_outputs(out64, n_act, a, lp, ent, v, 3, 0, f'probe {probe} n_act={n_act}')


@gpu
def test_policy_counters_under_graph_replay():
    """Both cleanrl.Policy step kinds captured in one CUDA graph: 128 features (pb_policy_mlp_sample, whose last CTA
    advances the counter) and 49 features (the packed forward, pb_sample_logits reading the counter on the device, then
    counter += 1).  Replay k draws at offset k: the actions match the restated draw (49 features: on the logits of an
    eager forward of the same x), the counters read k + 1 and the exit ticket is back at 0."""
    m = 1000
    pol_a = cleanrl.Policy(make_default(5, seed=1), fused_sample=True, seed=21)
    pol_b = cleanrl.Policy(make_default(6, seed=2, feats=49), fused_sample=True, seed=22)
    gen = torch.Generator(device=DEV).manual_seed(8)
    xa = torch.rand(m, 128, device=DEV, generator=gen) * 2 - 1
    xb = torch.rand(m, 49, device=DEV, generator=gen) * 2 - 1
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        pol_a(xa)
        pol_b(xb)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert pol_a._ticket is not None and pol_b._ticket is None
    pol_a._counter.zero_()
    pol_b._counter.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph):
        act_a, _, _, _ = pol_a(xa)
        act_b, _, _, _ = pol_b(xb)
    with torch.no_grad():
        w_cat, b_cat = pol_a.policy.head_matrix(cache=False)
        _, out64 = mlp_reference(xa, pol_a.policy.encoder.weight, pol_a.policy.encoder.bias, w_cat, b_cat)
        logits_b, _ = pol_b.policy(xb)
    probs_a, probs_b = softmax64(out64[:, :5]), softmax64(logits_b)
    for k in range(4):
        graph.replay()
        torch.cuda.synchronize()
        for name, acts, probs, seed, win in (('mlp kernel', act_a, probs_a, 21, WIN_MLP),
                                             ('sample_logits', act_b, probs_b, 22, WIN)):
            want, near = restated_draw(probs, uniforms(seed, k, m), win)
            bad = int(((want != cpu(acts)) & ~near).sum())
            assert bad == 0, (name, k, bad)
        assert int(pol_a._counter[0]) == k + 1 and int(pol_b._counter[0]) == k + 1
        assert int(pol_a._ticket[0]) == 0


# ---------------------------------------------------------------------------------------------------------------------
# the kernel samplers under a shifted head bias

SHIFT = 2.0 ** 20      # ulp 0.125: lse rounds to the 0.125 grid


def shifted_mismatches(prod, b_cat, n_act, acts, seed, offset):
    """Rows off the draw restated on the logits as the kernel forms them: fp32(head product) + fp32 bias, in fp32."""
    logits = prod[:, :n_act].float() + b_cat[:n_act].float()
    want, near = restated_draw(softmax64(logits), uniforms(seed, offset, acts.shape[0]), WIN_MLP)
    return int(((want != cpu(acts)) & ~near).sum())


@gpu
@pytest.mark.parametrize('n_act', [4, 10])
def test_policy_mlp_kernel_under_shifted_head_bias(n_act):
    """decoder.bias + 2^20 leaves the policy unchanged; pb_policy_mlp_sample's actions stay row-exact on all but at most
    1e-3 of the rows (those whose head product rounds across a 0.125 step)."""
    m = 65536
    net = make_default(n_act, seed=40 + n_act)
    with torch.no_grad():
        net.decoder.bias += SHIFT
    net.invalidate_cache()
    pol = cleanrl.Policy(net, fused_sample=True, seed=31)
    x = torch.rand(m, 128, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4)) * 2 - 1
    with torch.no_grad():
        a, _, _, _ = pol(x)
        w_cat, b_cat = net.head_matrix()
        prod, _ = mlp_reference(x, net.encoder.weight, net.encoder.bias, w_cat, b_cat)
    torch.cuda.synchronize()
    bad = shifted_mismatches(prod, b_cat, n_act, a, 31, 0)
    print(f'[policy-mlp, head bias + 2^20] n_act={n_act}: {bad} of {m} rows off the restated draw', flush=True)
    assert bad <= 1e-3 * m, bad


@gpu
@pytest.mark.parametrize('n_act', [4, 10])
def test_policy_lstm_kernel_under_shifted_head_bias(n_act):
    """The same for pb_policy_lstm_sample (cleanrl.RecurrentPolicy over LSTMWrapper(Default), 49 features)."""
    m = 65536
    pol = make_policy((49,), n_act, seed=13)
    net = pol.policy
    with torch.no_grad():
        net.policy.decoder.bias += SHIFT
    net.invalidate_cache()
    gen = torch.Generator(device=DEV).manual_seed(6)
    x = torch.rand(m, 49, device=DEV, generator=gen) * 2 - 1
    h0 = torch.randn(m, 128, device=DEV, generator=gen) * 0.5
    c0 = torch.randn(m, 128, device=DEV, generator=gen)
    h, c = h0.clone().unsqueeze(0), c0.clone().unsqueeze(0)
    with torch.no_grad():
        a, _, _, _, _ = pol(x, (h, c))
        h2, _, _ = reference_step(net, x, h0, c0)
        w_cat, b_cat = net.policy.head_matrix()
        prod = rna(h2) @ rna(w_cat).t()
    torch.cuda.synchronize()
    bad = shifted_mismatches(prod, b_cat, n_act, a, 13, 0)
    print(f'[policy-lstm, head bias + 2^20] n_act={n_act}: {bad} of {m} rows off the restated draw', flush=True)
    assert bad <= 1e-3 * m, bad
