"""models.Default with 8 to 15 actions on the hand-written kernels: the 16-row padded head matrix (n_act logit rows |
value row | zero rows, models.Default.head_matrix) through pb_ppo_loss's packed rows, pb_mlp_tail_backward_ex,
pb_pack_heads, pb_policy_mlp_sample and the _DefaultMLPUpdate chain of train()."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from test_gpu_experience import make_config
from test_gpu_mlp_tail import check_tail, tail, tail_inputs
from test_gpu_policy_lstm import fake_env
from test_gpu_ppo_loss import reference_loss

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')


def _loss_inputs(m, n_act, width, seed):
    torch.manual_seed(seed)
    out0 = torch.randn(m, width, device=DEV)
    out0[:, n_act + 1:] = 0
    actions = torch.randint(0, n_act, (m,), device=DEV)
    old_lp, adv, ret = -torch.rand(m, device=DEV) - 1, torch.randn(m, device=DEV), torch.randn(m, device=DEV)
    old_v = out0[:, n_act] + 0.15 * torch.randn(m, device=DEV)
    return out0, actions, old_lp, adv, ret, old_v


@pytest.mark.parametrize('m', [1, 4097, 100000])
@pytest.mark.parametrize('n_act', [8, 10, 15])
@pytest.mark.parametrize('clip_vloss', [True, False])
def test_ppo_loss_packed_rows_16(m, n_act, clip_vloss):
    """Packed [M, 16] rows: the loss and its gradient match the autograd formulation (tolerances of
    test_gpu_ppo_loss), the padding columns of the gradient are exactly 0 and every row is written whole."""
    cfg = pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=clip_vloss, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    out0, actions, old_lp, adv, ret, old_v = _loss_inputs(m, n_act, 16, m + n_act)
    a = out0.clone().requires_grad_(True)
    loss, st = clean_pufferl.fused_ppo_loss_packed(a, n_act, actions, old_lp, adv, ret, old_v, cfg)
    loss.backward()
    b = out0.clone().requires_grad_(True)
    ref, st_ref = reference_loss(b[:, :n_act], b[:, n_act:n_act + 1], actions, old_lp, adv, ret, old_v, cfg)
    ref.backward()
    assert torch.allclose(loss, ref, rtol=1e-5, atol=1e-6) and torch.allclose(st, st_ref, rtol=1e-5, atol=1e-6)
    assert float((a.grad - b.grad).abs().max()) <= 1e-5 * float(b.grad.abs().max()) + 1e-10
    assert float(a.grad[:, n_act + 1:].abs().sum()) == 0.0
    # the same call on a gradient buffer full of garbage: the kernel overwrites every column of every row
    grad = torch.full_like(out0, 7.0)
    stats = torch.empty(8, dtype=torch.float64, device=DEV)
    p = out0.data_ptr()
    _native.check(_native.lib().pb_ppo_loss(
        C.c_void_p(p), 16, C.c_void_p(p + 4 * n_act), 16, _native.ptr(actions), _native.ptr(old_lp), _native.ptr(adv),
        _native.ptr(ret), _native.ptr(old_v), m, n_act, C.c_float(0.1), int(clip_vloss), C.c_float(0.1), C.c_float(0.5),
        C.c_float(0.01), C.c_void_p(grad.data_ptr()), 16, C.c_void_p(grad.data_ptr() + 4 * n_act), 16,
        _native.ptr(stats), _native.stream_ptr()))
    assert torch.equal(grad, a.grad)


TAIL_HEADS = [(8, 1), (8, 4), (8, 7), (16, 8), (16, 15)]


@pytest.mark.parametrize('m', [1, 31, 32, 33, 37, 511, 512, 513, 4096, 524288 + 17])
@pytest.mark.parametrize('head_rows,n_act', TAIL_HEADS)
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_backward_matches_fp64(m, head_rows, n_act, strided):
    """pb_mlp_tail_backward_ex on 8-row (n_act <= 7) and 16-row heads vs fp64 torch on the same inputs: dPre, dW_heads,
    db_heads, db_enc within 1e-5 of each output's maximum (all fp32 FMA).  strided: dout rows head_rows + 4 floats apart
    take the generic kernel, contiguous [M, head_rows] rows the TMA-staged one.  M runs over the edges of its 32-row TMA
    chunks and 512-row CTAs; dPre and the gradients start as NaN, so a row the kernel skips fails.  The padding rows of
    dW_heads and db_heads are exactly 0."""
    hidden, dout, w = tail_inputs(m, 128, n_act, head_rows, m + n_act, strided)
    dpre, grads = tail(dout, w, hidden, head_rows)
    check_tail(dpre, grads, hidden, dout, w, head_rows, n_act)


@pytest.mark.parametrize('head_rows,n_act', [(8, 5), (16, 11)])
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_backward_small_launch_on_a_large_workspace(head_rows, n_act, strided):
    """A launch of 513 rows on the workspace a 524 305-row launch just filled with its per-CTA partials: the reduction
    reads only the small launch's own partials."""
    lib = _native.lib()
    big, small = 524288 + 17, 513
    ws = torch.empty(lib.pb_mlp_tail_workspace_bytes_ex(big, 128, head_rows), dtype=torch.uint8, device=DEV)
    for m in (big, small):
        hidden, dout, w = tail_inputs(m, 128, n_act, head_rows, m, strided)
        dpre, grads = tail(dout, w, hidden, head_rows, ws=ws)
    check_tail(dpre, grads, hidden, dout, w, head_rows, n_act)


@pytest.mark.parametrize('m', [37, 524288 + 17])
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_backward_ex_8_rows_is_the_existing_entry_point(m, strided):
    hidden, dout, w = tail_inputs(m, 128, 5, 8, 3, strided)
    a = tail(dout, w, hidden, 8)
    b = tail(dout, w, hidden, 8, legacy=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize('n_act', [8, 11, 15])
def test_pack_heads_16_rows_matches_head_matrix(n_act):
    torch.manual_seed(n_act)
    net = models.Default(fake_env((49,), n_act)).to(DEV)
    with torch.no_grad():
        for p in (net.decoder.bias, net.value_head.bias):
            p.uniform_(-1, 1)
    w_cat, b_cat = torch.full((16, 128), 9.0, device=DEV), torch.full((16,), 9.0, device=DEV)
    _native.check(_native.lib().pb_pack_heads(
        _native.ptr(net.decoder.weight), _native.ptr(net.decoder.bias), _native.ptr(net.value_head.weight),
        _native.ptr(net.value_head.bias), n_act, 128, _native.ptr(w_cat), _native.ptr(b_cat), None, None, 0,
        _native.stream_ptr()))
    ref_w, ref_b = net.head_matrix(cache=False)
    assert ref_w.shape == (16, 128)
    assert torch.equal(w_cat, ref_w) and torch.equal(b_cat, ref_b)


@pytest.mark.parametrize('n_act', [8, 10, 15])
@pytest.mark.parametrize('features', [128, 49, 1])
def test_default_16_row_fast_path_matches_plain_modules(n_act, features):
    """test_gpu_ppo_loss::test_default_mlp_fast_path_matches_plain_modules at 8 to 15 actions: the [M, 16] head GEMM and
    pb_mlp_tail_backward_ex(16) vs nn.Linear / relu, same tolerances."""
    check_fast_path_matches_plain_modules(features, n_act)


def check_fast_path_matches_plain_modules(features, n_act):
    """Default's fast path (forward_packed on [M, 8] or [M, 16] heads + pb_mlp_tail_backward_ex) vs the plain modules at
    M = 1, 37, 4096, 70001: outputs within 2e-3 (absolute and relative), each parameter gradient within 5e-3 of its
    largest entry.  -> (largest output error, largest gradient error / largest entry)."""
    torch.manual_seed(n_act + features)
    net = models.Default(fake_env((features,), n_act)).to(DEV)
    rows = 8 if n_act <= 7 else 16
    worst_out = worst_grad = 0.0
    for m in (1, 37, 4096, 70001):
        x = torch.randn(m, features, device=DEV)
        packed = net.forward_packed(x)
        assert packed is not None and packed[0].shape == (m, rows) and packed[1] == n_act
        g_logits, g_value = torch.randn(m, n_act, device=DEV), torch.randn(m, 1, device=DEV)
        grads = []
        for fast in (True, False):
            net.fast_path = fast
            net.zero_grad()
            logits, value = net(x)
            ((logits * g_logits).sum() + (value * g_value).sum()).backward()
            grads.append((logits.detach(), value.detach(), [p.grad.clone() for p in net.parameters()]))
        net.fast_path = True
        (l1, v1, g1), (l0, v0, g0) = grads
        assert torch.allclose(l1, l0, rtol=2e-3, atol=2e-3) and torch.allclose(v1, v0, rtol=2e-3, atol=2e-3)
        worst_out = max(worst_out, float((l1 - l0).abs().max()), float((v1 - v0).abs().max()))
        for a, b in zip(g1, g0):
            scale = float(b.abs().max()) + 1e-6
            assert float((a - b).abs().max()) <= 5e-3 * scale, (m, float((a - b).abs().max()), scale)
            worst_grad = max(worst_grad, float((a - b).abs().max()) / scale)
    print(f'[default-fast-path] F={features} n_act={n_act} rows={rows}: max output err {worst_out:.2e}, '
          f'max grad err / max {worst_grad:.2e}', flush=True)
    return worst_out, worst_grad


@pytest.mark.parametrize('n_act', [8, 10, 15])
@pytest.mark.parametrize('m', [1, 100, 16384, 20001])
def test_fused_policy_step_16_rows_matches_torch_policy(n_act, m):
    """pb_policy_mlp_sample with two n8 head blocks vs the torch modules (tolerances of
    test_gpu_ppo_loss::test_fused_policy_step_matches_torch_policy), actions in [0, n_act) following the softmax, and
    the device counter / exit ticket."""
    torch.manual_seed(1)
    net = models.Default(fake_env((128,), n_act)).to(DEV)
    with torch.no_grad():
        net.decoder.weight.mul_(30.0)
    pol = cleanrl.Policy(net, fused_sample=True, seed=5).to(DEV)
    x = torch.randn(m, 128, device=DEV)
    vr, lr = torch.zeros(m, device=DEV), torch.zeros(m, device=DEV)
    ar = torch.full((m,), -1, dtype=torch.int64, device=DEV)
    with torch.no_grad():
        a, lp, ent, v = pol(x, out=(vr, lr, ar))
        assert pol._ticket is not None            # the exit ticket exists only on the one-kernel step
        assert a.data_ptr() == ar.data_ptr() and v.data_ptr() == vr.data_ptr()
        net.fast_path = False
        _, ref_lp, ref_ent, ref_v = pol(x, action=ar)
        logits, _ = net(x)
        net.fast_path = True
    assert int(ar.min()) >= 0 and int(ar.max()) < n_act
    assert torch.allclose(lr, ref_lp, atol=3e-3), float((lr - ref_lp).abs().max())
    assert torch.allclose(ent, ref_ent, atol=3e-3) and torch.allclose(vr, ref_v.flatten(), atol=3e-3)
    if m >= 16384:
        freq = torch.bincount(ar, minlength=n_act).float() / m
        expect = torch.softmax(logits, -1).mean(0)
        assert float((freq - expect).abs().max()) < 0.02
    assert int(pol._counter.item()) == 1 and int(pol._ticket.item()) == 0
    with torch.no_grad():
        a2, _, _, _ = pol(x)
    assert int(pol._counter.item()) == 2 and int(pol._ticket.item()) == 0
    assert int(a2.min()) >= 0 and int(a2.max()) < n_act
    if m >= 16384:
        assert 0.3 < float((a2 != ar).float().mean()) < 0.95


def _train_run(env, n, h, manual, **kw):
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=7).cuda()
    data = clean_pufferl.create(make_config(n, h, env=env, manual_update=manual, **kw), vec, pol)
    return vec, pol, data


@pytest.mark.parametrize('env,n_act', [('squared', 8), ('bandit', 10)])
def test_manual_update_16_rows_matches_autograd_update(env, n_act):
    """test_gpu_optim::test_manual_update_matches_autograd_update on envs with 8 and 10 actions: the hand-written chain
    on 16-row heads (slabs, not the fused kernel) vs autograd + clip_grad_norm_ + torch.optim.Adam, same tolerances."""
    check_manual_update_matches_autograd(env, n_act)


def check_manual_update_matches_autograd(env, n_act):
    """train() on env through the hand-written chain on slabs (head_rows 8 for n_act <= 7, else 16) vs autograd +
    clip_grad_norm_ + torch.optim.Adam from the same seed and rollout: parameters within 2e-5, losses within 1e-4
    relative.  -> (largest parameter difference, largest loss difference)."""
    n, h = 64, 32
    rows = 8 if n_act <= 7 else 16
    params, losses, used, states = {}, {}, {}, {}
    for manual in (True, False):
        vec, pol, data = _train_run(env, n, h, manual)
        assert pol.policy.decoder.weight.shape[0] == n_act
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        params[manual] = [p.detach().cpu().clone() for p in pol.parameters()]
        losses[manual] = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy,
                                   data.losses.approx_kl, data.losses.clipfrac, data.losses.explained_variance])
        used[manual] = data.manual_update is not None
        if manual:
            assert data.train_minibatch_path == 'slabs' and data.manual_update.used_fused is False
            assert data.manual_update.head_rows == rows and data.manual_update.w_cat.shape == (rows, 128)
        states[manual] = [float(data.optimizer.state[p]['step']) for p in pol.parameters()]
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        assert np.isfinite(data.losses.policy_loss)
        clean_pufferl.close(data)
    assert used[True] and not used[False]
    assert states[True] == states[False] == [4.0] * 6
    diff = max(float((a - b).abs().max()) for a, b in zip(params[True], params[False]))
    lerr = float((np.abs(losses[True] - losses[False]) / (np.abs(losses[False]) + 1e-30)).max())
    print(f'[manual-update] {env} n_act={n_act} rows={rows}: param diff {diff:.2e}, largest relative loss diff '
          f'{lerr:.2e}', flush=True)
    assert diff <= 2e-5, diff
    assert np.allclose(losses[True], losses[False], rtol=1e-4, atol=1e-6), (losses[True], losses[False])
    return diff, lerr


@pytest.mark.parametrize('env', ['squared', 'bandit'])
def test_manual_update_16_rows_inside_train_graph(env):
    """The 16-row chain captured in the train graph replays to the parameters of eager execution (comparison of
    test_gpu_optim::test_fused_update_kernel_inside_train_graph)."""
    n, h = 128, 32
    out = {}
    for graph in (False, True):
        vec, pol, data = _train_run(env, n, h, True, cuda_graph_train=graph, cuda_graph_rollout=False)
        for _ in range(3):
            clean_pufferl.evaluate(data)
            clean_pufferl.train(data)
        assert data.manual_update is not None and data.manual_update.used_fused is False
        assert data.train_minibatch_path == 'slabs'
        assert (data.train_graph_state == 2) == graph
        out[graph] = torch.cat([p.detach().reshape(-1).cpu() for p in pol.parameters()])
        clean_pufferl.close(data)
    assert float((out[True] - out[False]).abs().max()) < 1e-4


def test_bandit_learns_on_the_hand_written_update():
    """10-arm bandit (tests/test_gpu_ocean_learning.py settings, seed 1, budget 20) learns through _DefaultMLPUpdate on
    16-row heads, captured in the train graph."""
    from test_gpu_ocean_learning import BUDGET, run_case
    first, history, record = run_case('bandit', seed=1, iters=BUDGET['bandit'])
    print(f'[bandit, 16-row heads] passed at iteration {first}; {record}; last metrics {history[-3:]}', flush=True)
    assert first is not None, (history, record)
    assert record['update'] == 'hand-written' and record['minibatch_form'] == 'slabs', record
    assert record['graph_state'] == 2, record
