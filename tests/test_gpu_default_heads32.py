"""models.Default with 16 to 31 actions on the hand-written kernels: the 32-row padded head matrix (n_act logit rows |
value row | zero rows, models.Default.head_matrix) through pb_ppo_loss's packed rows, pb_mlp_tail_backward_ex,
pb_pack_heads, pb_policy_mlp_sample's four n8 head blocks and the _DefaultMLPUpdate chain of train().
More than 31 actions keeps the plain modules; LSTMWrapper(Default) with more than 15 actions keeps the cuDNN path."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
import util_peer as up
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from test_gpu_default_heads16 import _loss_inputs
from test_gpu_default_hidden import make_default, policy_step_abi
from test_gpu_experience import make_config
from test_gpu_mlp_tail import check_tail, tail, tail_inputs
from test_gpu_peer_staged import Engine, TorchAdam, assert_same_bits, default_parameters, round4, step_gradients
from test_gpu_policy_lstm import fake_env
from test_gpu_ppo_loss import reference_loss
from test_gpu_sampling import G, SHIFT, TIE, check_mlp_outputs, mlp_reference, shifted_mismatches
from util_gpu import restated_draw, softmax64, uniforms

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
P = _native.ptr
ARMS = 24


# ---------------------------------------------------------------------------------------------------------------------
# packed loss

@pytest.mark.parametrize('m', [1, 4097, 100000])
@pytest.mark.parametrize('n_act', [16, 17, 24, 31])
@pytest.mark.parametrize('clip_vloss', [True, False])
def test_ppo_loss_packed_rows_32(m, n_act, clip_vloss):
    """Packed [M, 32] rows: the loss and its gradient match the autograd formulation (tolerances of test_gpu_ppo_loss),
    the padding columns of the gradient are exactly 0, and a gradient buffer full of garbage is overwritten whole."""
    cfg = pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=clip_vloss, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    out0, actions, old_lp, adv, ret, old_v = _loss_inputs(m, n_act, 32, m + n_act)
    a = out0.clone().requires_grad_(True)
    loss, st = clean_pufferl.fused_ppo_loss_packed(a, n_act, actions, old_lp, adv, ret, old_v, cfg)
    loss.backward()
    b = out0.clone().requires_grad_(True)
    ref, st_ref = reference_loss(b[:, :n_act], b[:, n_act:n_act + 1], actions, old_lp, adv, ret, old_v, cfg)
    ref.backward()
    assert torch.allclose(loss, ref, rtol=1e-5, atol=1e-6) and torch.allclose(st, st_ref, rtol=1e-5, atol=1e-6)
    assert float((a.grad - b.grad).abs().max()) <= 1e-5 * float(b.grad.abs().max()) + 1e-10
    assert float(a.grad[:, n_act + 1:].abs().sum()) == 0.0
    grad = torch.full_like(out0, 7.0)
    stats = torch.empty(8, dtype=torch.float64, device=DEV)
    p = out0.data_ptr()
    _native.check(_native.lib().pb_ppo_loss(
        C.c_void_p(p), 32, C.c_void_p(p + 4 * n_act), 32, P(actions), P(old_lp), P(adv), P(ret), P(old_v), m, n_act,
        C.c_float(0.1), int(clip_vloss), C.c_float(0.1), C.c_float(0.5), C.c_float(0.01), C.c_void_p(grad.data_ptr()), 32,
        C.c_void_p(grad.data_ptr() + 4 * n_act), 32, P(stats), _native.stream_ptr()))
    assert torch.equal(grad, a.grad)


# ---------------------------------------------------------------------------------------------------------------------
# tail backward

@pytest.mark.parametrize('m', [1, 31, 32, 33, 511, 512, 513, 4096, 524288 + 17])
@pytest.mark.parametrize('hid', [128, 256, 384, 512])
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_32_rows_matches_fp64(m, hid, strided):
    """pb_mlp_tail_backward_ex(head_rows=32) vs fp64 torch: dPre, dW_heads, db_enc, db_heads within 1e-5 of each output's
    maximum; dPre and the gradients start as NaN, so an entry no 64-column slice writes fails; the padding rows of dW_heads
    and db_heads are exactly 0.  Contiguous [M, 32] dOut takes the TMA-staged kernel, rows 36 floats apart the strided one.
    n_act = 16 + m % 16 runs over 16, 17 and 31."""
    n_act = 16 + m % 16
    hidden, dout, w = tail_inputs(m, hid, n_act, 32, m + hid, strided)
    dpre, grads = tail(dout, w, hidden, 32)
    check_tail(dpre, grads, hidden, dout, w, 32, n_act)


@pytest.mark.parametrize('hid', [128, 256, 384, 512])
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_32_rows_small_launch_on_a_large_workspace(hid, strided):
    """513 rows on the workspace a 524 305-row launch just filled: the reduction reads only the small launch's
    partials."""
    lib = _native.lib()
    big, small = 524288 + 17, 513
    ws = torch.empty(lib.pb_mlp_tail_workspace_bytes_ex(big, hid, 32), dtype=torch.uint8, device=DEV)
    for m in (big, small):
        hidden, dout, w = tail_inputs(m, hid, 24, 32, m, strided)
        dpre, grads = tail(dout, w, hidden, 32, ws=ws)
    check_tail(dpre, grads, hidden, dout, w, 32, 24)


def test_mlp_tail_other_head_rows_are_refused_before_any_launch():
    """head_rows 24 and 64 give PB_ERR_UNSUPPORTED before any launch, nothing written; the workspace size of 32 rows is
    the formula of the other row counts."""
    lib = _native.lib()
    m, hid = 100, 128
    assert lib.pb_mlp_tail_workspace_bytes_ex(m, hid, 32) == 1 * (32 * hid + hid + 32) * 4
    assert lib.pb_mlp_tail_workspace_bytes_ex(4096, 256, 32) == 8 * (32 * 256 + 256 + 32) * 4
    ws = torch.empty(lib.pb_mlp_tail_workspace_bytes_ex(m, hid, 32) * 4, dtype=torch.uint8, device=DEV)
    for rows in (24, 64):
        hidden = torch.ones(m, hid, device=DEV)
        dout, w = torch.ones(m, rows, device=DEV), torch.ones(rows, hid, device=DEV)
        dpre, grads = torch.full_like(hidden, 7.0), torch.full((rows * hid + hid + rows,), 7.0, device=DEV)
        torch.cuda.synchronize()
        l0 = lib.pb_launch_count()
        rc = lib.pb_mlp_tail_backward_ex(P(dout), rows, P(w), P(hidden), m, hid, P(dpre), P(grads), P(ws), ws.numel(),
                                         rows, _native.stream_ptr())
        assert rc == _native.PB_ERR_UNSUPPORTED and lib.pb_launch_count() == l0, (rows, rc)
        assert bool((dpre == 7.0).all()) and bool((grads == 7.0).all())


# ---------------------------------------------------------------------------------------------------------------------
# pack heads

@pytest.mark.parametrize('n_act', [16, 17, 24, 31])
@pytest.mark.parametrize('hid', [128, 256])
def test_pack_heads_32_rows_matches_head_matrix(n_act, hid):
    torch.manual_seed(n_act + hid)
    net = models.Default(fake_env((49,), n_act), hidden_size=hid).to(DEV)
    with torch.no_grad():
        for p in (net.decoder.bias, net.value_head.bias):
            p.uniform_(-1, 1)
    w_cat, b_cat = torch.full((32, hid), 9.0, device=DEV), torch.full((32,), 9.0, device=DEV)
    _native.check(_native.lib().pb_pack_heads(
        P(net.decoder.weight), P(net.decoder.bias), P(net.value_head.weight), P(net.value_head.bias), n_act, hid,
        P(w_cat), P(b_cat), None, None, 0, _native.stream_ptr()))
    ref_w, ref_b = net.head_matrix(cache=False)
    assert ref_w.shape == (32, hid)
    assert torch.equal(w_cat, ref_w) and torch.equal(b_cat, ref_b)


def test_head_matrix_rows():
    """8 rows up to 7 actions, 16 up to 15, 32 up to 31, then the next multiple of 8 (the plain path's width)."""
    for n_act, rows in ((1, 8), (7, 8), (8, 16), (15, 16), (16, 32), (23, 32), (31, 32), (32, 40), (40, 48)):
        net = models.Default(fake_env((3,), n_act))
        assert net.head_matrix(cache=False)[0].shape == (rows, 128), n_act


# ---------------------------------------------------------------------------------------------------------------------
# rollout step

def _policy_case(hid, n_act, m):
    """pb_policy_mlp_sample through the ABI on observation rows 132 floats apart (NaN past column 128), with G canary
    rows around each output and the counter preset to 2^33 + 5; checked against the fp64 restatement."""
    start = 2 ** 33 + 5
    net = make_default(hid, n_act, seed=m + n_act + hid)
    gen = torch.Generator(device=DEV).manual_seed(m * 31 + n_act)
    buf = torch.full((m + 2, 132), float('nan'), device=DEV)
    buf[1:m + 1, :128] = torch.rand(m, 128, device=DEV, generator=gen) * 2 - 1
    x = buf[1:m + 1, :128]
    counter = torch.tensor([start], dtype=torch.int64, device=DEV)
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    bufs = [torch.full((m + 2 * G,), 7.0, device=DEV) for _ in range(3)] + \
        [torch.full((m + 2 * G,), -7, dtype=torch.int64, device=DEV)]
    vbuf, lbuf, ebuf, abuf = bufs
    _native.check(policy_step_abi(net, x, 132, counter, ticket, abuf[G:G + m], lbuf[G:G + m], vbuf[G:G + m],
                                  ebuf[G:G + m], 4))
    torch.cuda.synchronize()
    with torch.no_grad():
        w_cat, b_cat = net.head_matrix(cache=False)
        assert w_cat.shape == (32, hid)
        _, out64 = mlp_reference(x, net.encoder.weight, net.encoder.bias, w_cat, b_cat)
    check_mlp_outputs(out64, n_act, abuf[G:G + m], lbuf[G:G + m], ebuf[G:G + m], vbuf[G:G + m], 4, start,
                      f'H={hid} m={m} n_act={n_act}')
    for b, fill in ((vbuf, 7.0), (lbuf, 7.0), (ebuf, 7.0), (abuf, -7)):
        assert bool((b[:G] == fill).all()) and bool((b[G + m:] == fill).all())
    assert int(counter[0]) == start + 1 and int(ticket[0]) == 0


@pytest.mark.parametrize('m', [1, 63, 64, 65, 16385])
@pytest.mark.parametrize('n_act', [16, 24, 31])
@pytest.mark.parametrize('hid', [128, 256, 512])
def test_policy_mlp_32_heads_matches_fp64(hid, n_act, m):
    """pb_policy_mlp_sample with four n8 head blocks vs rna(x) @ rna(W_enc)^T + b -> relu -> rna(h) @ rna(W_cat)^T + b_cat in
    fp64: value, logprob and entropy within 2e-4, actions row-exact off the 1e-4 windows, canary rows untouched, the
    counter advanced by one and the exit ticket back at 0."""
    _policy_case(hid, n_act, m)


@pytest.mark.parametrize('n_act', range(16, 32))
def test_policy_mlp_32_heads_every_action_count(n_act):
    """The same at H = 128 and 20001 rows for every action count of the 32-row heads."""
    _policy_case(128, n_act, 20001)


@pytest.mark.parametrize('hid', [128, 512])
def test_policy_mlp_32_heads_under_graph_replay(hid):
    """cleanrl.Policy's one-kernel step with 24 actions captured in a CUDA graph: replay k draws at counter offset k
    (actions row-exact off the windows), the counter reads k + 1 and the exit ticket is back at 0."""
    m, n_act = 1000, ARMS
    pol = cleanrl.Policy(make_default(hid, n_act, seed=1), fused_sample=True, seed=21)
    x = torch.rand(m, 128, device=DEV, generator=torch.Generator(device=DEV).manual_seed(8)) * 2 - 1
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        pol(x)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert pol._ticket is not None
    pol._counter.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph):
        acts, _, _, _ = pol(x)
    with torch.no_grad():
        w_cat, b_cat = pol.policy.head_matrix(cache=False)
        _, out64 = mlp_reference(x, pol.policy.encoder.weight, pol.policy.encoder.bias, w_cat, b_cat)
    probs = softmax64(out64[:, :n_act])
    for k in range(4):
        graph.replay()
        torch.cuda.synchronize()
        want, near = restated_draw(probs, uniforms(21, k, m), 1e-4)
        assert int(((want != acts.cpu().numpy()) & ~near).sum()) == 0, k
        assert int(pol._counter[0]) == k + 1 and int(pol._ticket[0]) == 0


@pytest.mark.parametrize('hid', [128, 256, 512])
def test_policy_mlp_32_heads_tf32_tie_in_the_fourth_block(hid):
    """30 actions: the value is head column 30, in the fourth n8 block.  The value row sits on the exact TF32 tie
    1 + 2^-11 and hidden unit hid - 128 + j of row j is 1 (W_enc = I on the last 128-unit chunk, x = I), so the value
    moves by >= 4.8e-4 (more than the 2e-4 bound) if the head operand of that block is rounded any other way than
    cvt.rna.  At H > 128 the head columns come from the last ring stage."""
    m, n_act = 128, 30
    torch.manual_seed(hid)
    net = models.Default(fake_env((128,), n_act), hidden_size=hid).to(DEV)
    eye = torch.eye(128, device=DEV)
    with torch.no_grad():
        net.encoder.weight.zero_()
        net.encoder.weight[hid - 128:] = eye
        net.encoder.bias.zero_()
        net.decoder.weight.normal_(0, 0.5)
        net.decoder.bias.uniform_(-1, 1)
        net.value_head.weight.fill_(TIE)
        net.value_head.bias.zero_()
    net.invalidate_cache()
    pol = cleanrl.Policy(net, fused_sample=True, seed=3)
    with torch.no_grad():
        a, lp, ent, v = pol(eye)
        w_cat, b_cat = net.head_matrix()
        _, out64 = mlp_reference(eye, net.encoder.weight, net.encoder.bias, w_cat, b_cat)
    torch.cuda.synchronize()
    trunc = lambda t: (t.detach().float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32).double()  # noqa
    h_t = torch.relu(trunc(eye) @ trunc(net.encoder.weight).t() + net.encoder.bias.double())
    v_trunc = (trunc(h_t) @ trunc(w_cat).t() + b_cat.double())[:, n_act]
    assert float((out64[:, n_act] - v_trunc).abs().min()) >= 4.8e-4
    check_mlp_outputs(out64, n_act, a, lp, ent, v, 3, 0, f'fourth-block tie H={hid}')


@pytest.mark.parametrize('hid', [128, 256])
def test_policy_mlp_32_heads_under_shifted_head_bias(hid):
    """decoder.bias + 2^20 with 24 actions: the actions stay row-exact on all but at most 1e-3 of the rows (those whose
    head product rounds across a 0.125 step), as test_gpu_sampling checks for 8 and 16 head rows."""
    m = 65536
    net = make_default(hid, ARMS, seed=40 + hid)
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
    bad = shifted_mismatches(prod, b_cat, ARMS, a, 31, 0)
    print(f'[policy-mlp, 32 heads, head bias + 2^20] H={hid}: {bad} of {m} rows off the restated draw', flush=True)
    assert bad <= 1e-3 * m, bad


def test_more_than_31_actions_are_refused_and_keep_the_plain_path():
    """pb_policy_mlp_sample refuses n_act = 32 (PB_ERR_UNSUPPORTED, nothing launched or written) and pb_pack_heads
    n_act = 32; models.Default with 32 actions keeps nn.Linear, cleanrl.Policy the library sampler."""
    lib = _native.lib()
    m = 100
    net = make_default(128, 32)
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    acts = torch.full((m,), -7, dtype=torch.int64, device=DEV)
    lp, val, ent = (torch.full((m,), 7.0, device=DEV) for _ in range(3))
    x = torch.zeros(m, 128, device=DEV)
    torch.cuda.synchronize()
    l0 = lib.pb_launch_count()
    rc = policy_step_abi(net, x, 128, counter, ticket, acts, lp, val, ent, 1)
    assert rc == _native.PB_ERR_UNSUPPORTED and lib.pb_launch_count() == l0, rc
    assert int(counter[0]) == 0 and bool((acts == -7).all()) and bool((lp == 7.0).all())
    w_cat, b_cat = torch.zeros(40, 128, device=DEV), torch.zeros(40, device=DEV)
    rc = lib.pb_pack_heads(P(net.decoder.weight), P(net.decoder.bias), P(net.value_head.weight), P(net.value_head.bias),
                           32, 128, P(w_cat), P(b_cat), None, None, 0, _native.stream_ptr())
    assert rc == _native.PB_ERR_INVALID and lib.pb_launch_count() == l0, rc
    assert not net._fast_ok(x) and net.forward_packed(x) is None
    pol = cleanrl.Policy(net, fused_sample=True, seed=1)
    with torch.no_grad():
        assert pol._policy_step_fused(x) is None
        logits, value = net(x)
    assert logits.shape == (m, 32) and value.shape == (m, 1)


# ---------------------------------------------------------------------------------------------------------------------
# the fast path

@pytest.mark.parametrize('features', [128, 49, 1])
@pytest.mark.parametrize('n_act', [16, 24, 31])
@pytest.mark.parametrize('hid', [128, 256])
def test_default_32_row_fast_path_matches_plain_modules(features, n_act, hid):
    """Default's fast path ([M, 32] head GEMM + pb_mlp_tail_backward_ex(32)) vs the plain modules at M = 1, 37, 4096,
    70001: outputs within 2e-3, each parameter gradient within 5e-3 of its largest entry."""
    torch.manual_seed(n_act + features + hid)
    net = models.Default(fake_env((features,), n_act), hidden_size=hid).to(DEV)
    for m in (1, 37, 4096, 70001):
        x = torch.randn(m, features, device=DEV)
        packed = net.forward_packed(x)
        assert packed is not None and packed[0].shape == (m, 32) and packed[1] == n_act
        g_logits, g_value = torch.randn(m, n_act, device=DEV), torch.randn(m, 1, device=DEV)
        res = []
        for fast in (True, False):
            net.fast_path = fast
            net.zero_grad()
            logits, value = net(x)
            ((logits * g_logits).sum() + (value * g_value).sum()).backward()
            res.append((logits.detach(), value.detach(), [p.grad.clone() for p in net.parameters()]))
        net.fast_path = True
        (l1, v1, g1), (l0, v0, g0) = res
        assert torch.allclose(l1, l0, rtol=2e-3, atol=2e-3) and torch.allclose(v1, v0, rtol=2e-3, atol=2e-3)
        for a, b in zip(g1, g0):
            scale = float(b.abs().max()) + 1e-6
            assert float((a - b).abs().max()) <= 5e-3 * scale, (m, float((a - b).abs().max()), scale)


# ---------------------------------------------------------------------------------------------------------------------
# train()

def bandit_run(n, h, manual, monkeypatch=None, plans=None, arms=ARMS, **kw):
    if plans is not None:
        plan_fn = clean_pufferl.update_plan
        monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(plan_fn(d)) or plans[-1])
    vec = pvec.make(ocean.env_creator('bandit'), env_kwargs=dict(num_actions=arms), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=7).cuda()
    data = clean_pufferl.create(make_config(n, h, env='bandit', manual_update=manual, **kw), vec, pol)
    return vec, pol, data


def test_manual_update_32_rows_matches_autograd_update(monkeypatch):
    """train() on the 24-arm bandit through the hand-written chain on 32-row heads vs autograd + clip_grad_norm_ +
    torch.optim.Adam from the same seed and rollout: parameters within 2e-5, losses within 1e-4 relative, the Adam steps
    counted alike.  The plan is ('mlp_chain', 'slabs')."""
    n, h = 64, 32
    params, losses, states = {}, {}, {}
    for manual in (True, False):
        plans = []
        vec, pol, data = bandit_run(n, h, manual, monkeypatch, plans)
        assert pol.policy.decoder.weight.shape[0] == ARMS
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        params[manual] = [p.detach().cpu().clone() for p in pol.parameters()]
        losses[manual] = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy,
                                   data.losses.approx_kl, data.losses.clipfrac, data.losses.explained_variance])
        if manual:
            assert (plans[-1].engine, plans[-1].form) == ('mlp_chain', 'slabs'), plans[-1]
            mu = data.manual_update
            assert mu.head_rows == 32 and mu.w_cat.shape == (32, 128) and mu.used_fused is False
            assert mu.gflat.numel() == 128 * 1 + 32 * 128 + 128 + 32
        else:
            assert data.manual_update is None
        states[manual] = [float(data.optimizer.state[p]['step']) for p in pol.parameters()]
        clean_pufferl.close(data)
    assert states[True] == states[False]
    diff = max(float((a - b).abs().max()) for a, b in zip(params[True], params[False]))
    print(f'[manual-update] bandit {ARMS} arms rows=32: param diff {diff:.2e}', flush=True)
    assert diff <= 2e-5, diff
    assert np.allclose(losses[True], losses[False], rtol=1e-4, atol=1e-6), (losses[True], losses[False])


@pytest.mark.parametrize('n_act', [16, 31])
def test_manual_update_32_rows_on_128_features_matches_autograd(n_act):
    """_DefaultMLPUpdate on a synthetic 128-feature minibatch ([2, 2048, 128] slabs, three optimizer steps) vs nn.Linear
    + the reference loss + autograd + clip_grad_norm_ + torch.optim.Adam on a copy of the model: loss statistics within
    1e-4 relative; parameters within 2e-5 but for at most 1 in 1000 entries, which stay within 2 lr per step.  Adam's
    first steps move an entry by about lr whatever the size of its gradient, so an entry whose gradient over random
    observations cancels down to fp32 rounding noise may step the other way in one of the two runs (the bound of
    test_gpu_default_hidden::test_manual_update_matches_autograd_update)."""
    torch.manual_seed(n_act)
    cfg = make_config(64, 32)
    model = models.Default(fake_env((128,), n_act)).to(DEV)
    with torch.no_grad():
        model.decoder.weight.mul_(20.0)
    ref = copy.deepcopy(model)
    ref.fast_path = False
    opt = torch.optim.Adam(model.parameters(), lr=cfg.learning_rate, eps=1e-5, fused=True)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=cfg.learning_rate, eps=1e-5, fused=True)
    data = pufferlib_b200.namespace(policy=pufferlib_b200.namespace(policy=model), optimizer=opt, config=cfg)
    mu = clean_pufferl._DefaultMLPUpdate(data)
    assert mu.head_rows == 32
    lerr = 0.0
    for step in range(3):
        g_, r_ = 2, 2048
        m = g_ * r_
        x = torch.randn(g_, r_, 128, device=DEV)
        with torch.no_grad():
            logits, value = ref(x.view(m, 128))
            act = torch.distributions.Categorical(logits=logits).sample()
            _, lp, _ = cleanrl.sample_logits(logits, act)
        olp = lp + 0.1 * torch.randn(m, device=DEV)
        adv, ret = torch.randn(m, device=DEV), torch.randn(m, device=DEV)
        oval = value.view(-1) + 0.1 * torch.randn(m, device=DEV)
        mb = pufferlib_b200.namespace(obs=x, slab_form=True, actions=act, logprobs=olp, values=oval, advantages=adv,
                                      returns=ret, row_slab_stride=None, adv_norm=None)
        mu.pack_heads()
        mu.forward_backward(0, 1, mb, cfg)
        mu.optimizer_step(cfg)
        got = mu.loss_means(1)
        ref_opt.zero_grad()
        logits, value = ref(x.view(m, 128))
        loss, st = reference_loss(logits, value, act, olp, adv, ret, oval, cfg)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), cfg.max_grad_norm)
        ref_opt.step()
        assert torch.allclose(got, st, rtol=1e-4, atol=1e-6), (step, got, st)
        lerr = max(lerr, float(((got - st).abs() / (st.abs() + 1e-30)).max()))
    d = torch.cat([(a - b).detach().abs().reshape(-1) for a, b in zip(model.parameters(), ref.parameters())])
    print(f'[manual-update] 128 features n_act={n_act} rows=32: param diff {float(d.max()):.2e}, entries past 2e-5 '
          f'{int((d > 2e-5).sum())} of {d.numel()}, loss diff {lerr:.2e}', flush=True)
    assert float(d.max()) <= 2 * cfg.learning_rate * 3, float(d.max())
    assert int((d > 2e-5).sum()) <= d.numel() // 1000, int((d > 2e-5).sum())


def test_manual_update_32_rows_inside_train_graph(monkeypatch):
    """The 32-row chain captured whole in the train graph replays to the parameters of eager execution (within 1e-4);
    the plan is ('mlp_chain', 'slabs', 'whole')."""
    n, h = 128, 32
    out = {}
    for graph in (False, True):
        plans = []
        vec, pol, data = bandit_run(n, h, True, monkeypatch, plans, cuda_graph_train=graph, cuda_graph_rollout=False)
        for _ in range(3):
            clean_pufferl.evaluate(data)
            clean_pufferl.train(data)
        p = plans[-1]
        assert (p.engine, p.form, p.capture) == ('mlp_chain', 'slabs', 'whole' if graph else None), p
        assert data.manual_update.head_rows == 32 and (data.train_graph_state == 2) == graph
        out[graph] = torch.cat([q.detach().reshape(-1).cpu() for q in pol.parameters()])
        clean_pufferl.close(data)
    assert float((out[True] - out[False]).abs().max()) < 1e-4


@pytest.mark.parametrize('features', [128, 1])
@pytest.mark.parametrize('world,rank', [(2, 1), (4, 0), (8, 7)])
def test_clip_adam_peer_on_the_32_row_buffer(world, rank, features):
    """pb_clip_adam_peer (the chain's optimizer step on several ranks) on _DefaultMLPUpdate's 32-row flat buffer
    dW_enc | 32 head rows x 128 | db_enc | 32 head biases, against staged peers (tests/util_peer.py), five steps: bitwise
    pb_clip_adam on the rank-order sum, and torch within test_gpu_peer_staged's bounds."""
    n_act, hid = ARMS, 128
    w_cat, b_enc, b_cat = hid * features, hid * features + 32 * hid, hid * features + 33 * hid
    n = b_cat + 32
    assert n % 4 == 0
    views = [(0, hid * features), (b_enc, hid), (w_cat, n_act * hid), (b_cat, n_act), (w_cat + n_act * hid, hid),
             (b_cat + n_act, 1)]
    torch.manual_seed(7)
    lib, s = _native.lib(), _native.stream_ptr()
    params = default_parameters(features, n_act, DEV)
    fused, plain = Engine(params, n, views, n_act, DEV), Engine(params, n, views, n_act, DEV)
    ref = TorchAdam(params, views, world, None)
    peers = up.StagedPeers(world, rank, round4(n), DEV, sliced=False)
    for it, g in enumerate(step_gradients(n, views, world, 100 * features + n_act, DEV)):
        summed = up.rank_order_sum(g)
        fused.flat.copy_(g[rank])
        peers.exchange(fused.flat, g, lambda comm: _native.check(lib.pb_clip_adam_peer(
            fused.arr, 6, *fused.hyper(world, None), C.byref(comm), P(fused.flat), n, s)))
        plain.flat.copy_(summed)
        _native.check(lib.pb_clip_adam(plain.arr, 6, *plain.hyper(world, None), s))
        norm = ref.step(summed)
        peers.check_epoch()
        peers.check_buffers()
        assert torch.equal(up.bits(fused.flat), up.bits(summed))
        assert_same_bits(fused, plain, f'step {it}, pb_clip_adam_peer vs pb_clip_adam on the sum')
        ref.check(fused, norm, it)


def test_lstm_default_with_24_actions_trains_on_cudnn():
    """RecurrentPolicy(LSTMWrapper(Default)) with 24 actions and fused_update=True: the fused recurrent kernels take at
    most 15 actions, so evaluate runs the library step and train() the cuDNN path, with finite losses."""
    n, h = 128, 32
    vec = pvec.make(ocean.env_creator('bandit'), env_kwargs=dict(num_actions=ARMS), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    env = vec.driver_env
    net = models.LSTMWrapper(env, models.Default(env), input_size=128, hidden_size=128)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=3, fused_update=True).cuda()
    data = clean_pufferl.create(make_config(n, h, env='bandit'), vec, pol)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        assert data.train_recurrent_path == 'cudnn' and data.manual_update is None
        assert np.isfinite(data.losses.policy_loss) and np.isfinite(data.losses.value_loss)
    clean_pufferl.close(data)


# iterations (evaluate + train) allowed for the 24-arm bandit: >= 2x the worst of seeds 1, 2, 3 on an H100 (DESIGN.md §4)
BANDIT24_BUDGET = 24


@pytest.mark.parametrize('seed', [1, 2, 3])
def test_bandit_24_arms_learns_on_the_hand_written_update(seed):
    """The 24-arm bandit (tests/test_gpu_ocean_learning.py settings) pulls its winning arm at least 90 % of the time within
    BANDIT24_BUDGET iterations, on the 32-row kernels: the one-kernel rollout step is not reached (1 feature), the
    fast-path forward and the hand-written chain captured in the train graph are."""
    from test_gpu_ocean_learning import N, make_config as ocean_config
    arm = int(np.random.RandomState(42).randint(0, ARMS))       # the reference env's winning arm
    torch.manual_seed(seed)
    vec = pvec.make(ocean.env_creator('bandit'), env_kwargs=dict(num_actions=ARMS), num_envs=N, backend=pvec.B200)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=seed).cuda()
    data = clean_pufferl.create(ocean_config(seed=seed), vec, pol)
    history = []
    for _ in range(BANDIT24_BUDGET):
        clean_pufferl.evaluate(data)
        history.append(float((data.experience.actions == arm).float().mean()))
        if history[-1] >= 0.9:
            break
        clean_pufferl.train(data)
        assert data.manual_update is not None and data.manual_update.head_rows == 32
        assert data.train_minibatch_path == 'slabs' and data.train_graph_state in (1, 2)
    clean_pufferl.close(data)
    print(f'[bandit, {ARMS} arms, seed {seed}] {len(history)} rollouts; last shares {history[-3:]}', flush=True)
    assert history[-1] >= 0.9, history
