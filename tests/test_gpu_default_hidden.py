"""models.Default with 256, 384 and 512 hidden units on the hand-written kernels: pb_policy_mlp_sample's chunked
rollout step (the W_enc ring of k_policy_mlp_sample), pb_mlp_tail_backward_ex over 128-column slices of the hidden layer (both the
TMA-staged and the strided kernel), the fast-path forward / backward, and the _DefaultMLPUpdate chain of train().
The H = 128 kernels are covered by test_gpu_sampling, test_gpu_default_heads16 and test_gpu_ppo_loss."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from test_gpu_experience import make_config
from test_gpu_mlp_tail import check_tail, tail, tail_inputs
from test_gpu_policy_lstm import fake_env
from test_gpu_sampling import G, TIE, check_mlp_outputs, mlp_reference
from util_gpu import restated_draw, softmax64, uniforms

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
P = _native.ptr
WIDE = (256, 384, 512)


def make_default(hid, n_act, seed=0, feats=128):
    torch.manual_seed(seed)
    net = models.Default(fake_env((feats,), n_act), hidden_size=hid).to(DEV)
    with torch.no_grad():            # informative heads: the 0.01-std init gives near-uniform policies
        net.decoder.weight.mul_(20.0)
        net.decoder.bias.uniform_(-1, 1)
    net.invalidate_cache()
    return net


# ---------------------------------------------------------------------------------------------------------------------
# rollout step

def policy_step_abi(net, x, stride, counter, ticket, acts, lp, val, ent, seed, hid=None, feats=128):
    w_cat, b_cat = net.head_matrix(cache=False)
    w_enc = models._round_tf32(net.encoder.weight)
    return _native.lib().pb_policy_mlp_sample(
        P(x), stride, P(w_enc), P(net.encoder.bias), P(w_cat), P(b_cat), x.shape[0], feats,
        hid or net.encoder.weight.shape[0], net.decoder.weight.shape[0], C.c_uint64(seed), P(counter), P(ticket), P(acts),
        P(lp), P(val), P(ent), _native.stream_ptr())


@pytest.mark.parametrize('m', [1, 63, 64, 65, 16385])
@pytest.mark.parametrize('n_act', [1, 4, 7, 8, 15])
@pytest.mark.parametrize('hid', WIDE)
def test_policy_mlp_wide_matches_fp64(hid, n_act, m):
    """pb_policy_mlp_sample at H = 256, 384, 512 vs rna(x) @ rna(W_enc)^T + b -> relu -> rna(h) @ rna(W_cat)^T + b_cat in
    fp64: value, logprob and entropy within 2e-4 (the H = 128 bound: the restatement carries every TF32 rounding, what
    is left is fp32 accumulation over H + 128 products), actions row-exact off the 1e-4 windows.  Observation rows are
    132 floats apart with NaN in the 4 columns past 128; G canary rows before and after each output stay untouched; the
    draw uses the preset counter 2^33 + 5, which the last CTA advances by one, and the ticket is back at 0."""
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
        _, out64 = mlp_reference(x, net.encoder.weight, net.encoder.bias, w_cat, b_cat)
    check_mlp_outputs(out64, n_act, abuf[G:G + m], lbuf[G:G + m], ebuf[G:G + m], vbuf[G:G + m], 4, start,
                      f'H={hid} m={m} n_act={n_act}')
    for b, fill in ((vbuf, 7.0), (lbuf, 7.0), (ebuf, 7.0), (abuf, -7)):
        assert bool((b[:G] == fill).all()) and bool((b[G + m:] == fill).all())
    assert int(counter[0]) == start + 1 and int(ticket[0]) == 0


@pytest.mark.parametrize('hid', [256, 512])
def test_policy_mlp_wide_under_graph_replay(hid):
    """cleanrl.Policy's one-kernel step at H > 128 captured in a CUDA graph: replay k draws at counter offset k (actions
    row-exact off the windows), the counter reads k + 1 and the exit ticket is back at 0."""
    m, n_act = 1000, 5
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


@pytest.mark.parametrize('n_act', [3, 10])
def test_policy_mlp_wide_tf32_tie_in_second_chunk(n_act):
    """H = 256 with x = 0 and b_enc = 1 + 2^-11 (an exact TF32 tie) on units 128..255 only: relu(h) is the tie in the
    second chunk and 0 in the first, so the value moves by >= 4.8e-4 (more than the 2e-4 bound) if the second chunk
    rounds relu(h) any other way than cvt.rna.  n_act 3 and 10 take the 8- and 16-row heads."""
    m, hid = 64, 256
    net = make_default(hid, n_act, seed=n_act)
    with torch.no_grad():
        net.encoder.bias.zero_()
        net.encoder.bias[128:] = TIE
        net.decoder.weight.normal_(0, 0.05)
        net.value_head.weight.fill_(1.0 / 128)
        net.value_head.bias.zero_()
    net.invalidate_cache()
    x = torch.zeros(m, 128, device=DEV)
    pol = cleanrl.Policy(net, fused_sample=True, seed=3)
    with torch.no_grad():
        a, lp, ent, v = pol(x)
        w_cat, b_cat = net.head_matrix()
        _, out64 = mlp_reference(x, net.encoder.weight, net.encoder.bias, w_cat, b_cat)
    torch.cuda.synchronize()
    trunc = lambda t: (t.detach().float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32).double()  # noqa
    h_t = torch.relu(net.encoder.bias.double()).expand(m, hid)
    v_trunc = (trunc(h_t) @ trunc(w_cat).t() + b_cat.double())[:, n_act]
    assert float((out64[:, n_act] - v_trunc).abs().min()) >= 4.8e-4        # the probe separates the roundings
    check_mlp_outputs(out64, n_act, a, lp, ent, v, 3, 0, f'second-chunk tie n_act={n_act}')


@pytest.mark.parametrize('n_act', [5, 12, 24])
@pytest.mark.parametrize('hid', WIDE)
def test_policy_mlp_wide_zero_units_match_hidden_128(hid, n_act):
    """Every hidden size runs one arithmetic: a Default at H = 256, 384, 512 whose encoder rows, encoder bias and head
    columns past unit 128 are zero gives, bit for bit, the actions, logprobs, values, entropies, counter and ticket of the
    H = 128 Default made of its first 128 units (the extra chunks add exact zeros).  n_act 5, 12, 24 take the 8-, 16- and
    32-row heads; 20001 rows end in a partial CTA; observation rows are 132 floats apart."""
    m, start, seed = 20001, 2 ** 33 + 5, 9
    wide = make_default(hid, n_act, seed=hid + n_act)
    narrow = make_default(128, n_act)
    with torch.no_grad():
        wide.encoder.weight[128:] = 0
        wide.encoder.bias[128:] = 0
        wide.decoder.weight[:, 128:] = 0
        wide.value_head.weight[:, 128:] = 0
        for a, b in ((narrow.encoder.weight, wide.encoder.weight[:128]), (narrow.encoder.bias, wide.encoder.bias[:128]),
                     (narrow.decoder.weight, wide.decoder.weight[:, :128]), (narrow.decoder.bias, wide.decoder.bias),
                     (narrow.value_head.weight, wide.value_head.weight[:, :128]),
                     (narrow.value_head.bias, wide.value_head.bias)):
            a.copy_(b)
    wide.invalidate_cache()
    narrow.invalidate_cache()
    x = (torch.rand(m, 132, device=DEV, generator=torch.Generator(device=DEV).manual_seed(n_act)) * 2 - 1)[:, :128]
    outs = []
    for net in (wide, narrow):
        counter = torch.tensor([start], dtype=torch.int64, device=DEV)
        ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
        acts = torch.full((m,), -7, dtype=torch.int64, device=DEV)
        lp, val, ent = (torch.full((m,), 7.0, device=DEV) for _ in range(3))
        _native.check(policy_step_abi(net, x, 132, counter, ticket, acts, lp, val, ent, seed))
        outs.append((acts, lp, val, ent, counter, ticket))
    torch.cuda.synchronize()
    assert int(outs[0][4][0]) == start + 1
    for name, a, b in zip(('actions', 'logprobs', 'values', 'entropies', 'counter', 'ticket'), *outs):
        assert torch.equal(a, b), f'H={hid} n_act={n_act}: {name} differs from the H = 128 model'


# ---------------------------------------------------------------------------------------------------------------------
# tail backward

@pytest.mark.parametrize('m', [1, 31, 32, 33, 511, 512, 513, 4096, 524288 + 17])
@pytest.mark.parametrize('rows,n_act', [(8, 5), (16, 12)])
@pytest.mark.parametrize('hid', WIDE)
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_slices_match_fp64(m, rows, n_act, hid, strided):
    """pb_mlp_tail_backward_ex at H = 256, 384 and 512 vs fp64 torch: dPre, dW_heads, db_enc, db_heads within 1e-5 of
    each output's maximum; dPre and the gradients start as NaN, so an entry no slice writes fails; the padding rows of
    dW_heads and db_heads are exactly 0.  M runs over the edges of the 32-row TMA chunks and the 512-row CTAs."""
    hidden, dout, w = tail_inputs(m, hid, n_act, rows, m + hid, strided)
    dpre, grads = tail(dout, w, hidden, rows)
    check_tail(dpre, grads, hidden, dout, w, rows, n_act)


@pytest.mark.parametrize('rows,n_act', [(8, 5), (16, 11)])
@pytest.mark.parametrize('hid', WIDE)
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_slices_small_launch_on_a_large_workspace(rows, n_act, hid, strided):
    """513 rows on the workspace a 524 305-row launch just filled: the reduction reads only the small launch's
    partials."""
    lib = _native.lib()
    big, small = 524288 + 17, 513
    ws = torch.empty(lib.pb_mlp_tail_workspace_bytes_ex(big, hid, rows), dtype=torch.uint8, device=DEV)
    for m in (big, small):
        hidden, dout, w = tail_inputs(m, hid, n_act, rows, m, strided)
        dpre, grads = tail(dout, w, hidden, rows, ws=ws)
    check_tail(dpre, grads, hidden, dout, w, rows, n_act)


# ---------------------------------------------------------------------------------------------------------------------
# refusals

def test_other_hidden_sizes_are_refused_before_any_launch():
    """H = 192 and 640 give PB_ERR_UNSUPPORTED from pb_policy_mlp_sample and pb_mlp_tail_backward_ex, and in_features
    other than 128 from pb_policy_mlp_sample; nothing is launched and no output is written.  models.Default with 192
    hidden units keeps the plain modules."""
    lib = _native.lib()
    m = 100
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    ticket = torch.zeros(1, dtype=torch.int32, device=DEV)
    acts = torch.full((m,), -7, dtype=torch.int64, device=DEV)
    lp, val, ent = (torch.full((m,), 7.0, device=DEV) for _ in range(3))
    for hid, feats in ((192, 128), (640, 128), (256, 64), (256, 129), (128, 49)):
        net = make_default(hid, 4)
        x = torch.zeros(m, 132, device=DEV)
        torch.cuda.synchronize()
        l0 = lib.pb_launch_count()
        rc = policy_step_abi(net, x, 132, counter, ticket, acts, lp, val, ent, 1, hid=hid, feats=feats)
        assert rc == _native.PB_ERR_UNSUPPORTED and lib.pb_launch_count() == l0, (hid, feats, rc)
    for hid in (192, 640):
        for rows in (8, 16):
            hidden = torch.ones(m, hid, device=DEV)
            dout, w = torch.ones(m, rows, device=DEV), torch.ones(rows, hid, device=DEV)
            dpre, grads = torch.full_like(hidden, 7.0), torch.full((rows * hid + hid + rows,), 7.0, device=DEV)
            ws = torch.empty(lib.pb_mlp_tail_workspace_bytes_ex(m, hid, rows), dtype=torch.uint8, device=DEV)
            torch.cuda.synchronize()
            l0 = lib.pb_launch_count()
            rc = lib.pb_mlp_tail_backward_ex(P(dout), rows, P(w), P(hidden), m, hid, P(dpre), P(grads), P(ws), ws.numel(),
                                             rows, _native.stream_ptr())
            assert rc == _native.PB_ERR_UNSUPPORTED and lib.pb_launch_count() == l0, (hid, rows, rc)
            assert bool((dpre == 7.0).all()) and bool((grads == 7.0).all())
    assert int(counter[0]) == 0 and int(ticket[0]) == 0 and bool((acts == -7).all()) and bool((lp == 7.0).all())
    assert bool((val == 7.0).all()) and bool((ent == 7.0).all())
    net = make_default(192, 4, feats=49)
    x = torch.randn(37, 49, device=DEV)
    assert not net._fast_ok(x) and net.forward_packed(x) is None
    pol = cleanrl.Policy(make_default(192, 4), fused_sample=True, seed=1)
    with torch.no_grad():
        assert pol._policy_step_fused(torch.randn(37, 128, device=DEV)) is None
        logits, value = net(x)
    assert logits.shape == (37, 4) and value.shape == (37, 1)


# ---------------------------------------------------------------------------------------------------------------------
# the fast path and train()

@pytest.mark.parametrize('features', [128, 49, 1])
@pytest.mark.parametrize('hid', [256, 512])
def test_fast_path_matches_plain_modules(features, hid):
    """Default's fast path (forward_packed + pb_mlp_tail_backward_ex over slices) vs the plain modules at M = 1, 37,
    4096, 70001 and n_act 5: outputs within 2e-3, each parameter gradient within 5e-3 of its largest entry."""
    n_act = 5
    torch.manual_seed(features + hid)
    net = models.Default(fake_env((features,), n_act), hidden_size=hid).to(DEV)
    for m in (1, 37, 4096, 70001):
        x = torch.randn(m, features, device=DEV)
        packed = net.forward_packed(x)
        assert packed is not None and packed[0].shape == (m, 8)
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


def train_run(env, n, h, hid, manual, monkeypatch=None, plans=None, **kw):
    if plans is not None:
        plan_fn = clean_pufferl.update_plan
        monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(plan_fn(d)) or plans[-1])
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env, hidden_size=hid), fused_sample=True, seed=7).cuda()
    data = clean_pufferl.create(make_config(n, h, env=env, manual_update=manual, **kw), vec, pol)
    return vec, pol, data


@pytest.mark.parametrize('hid', [256, 512])
@pytest.mark.parametrize('env', ['squared', 'breakout'])
def test_manual_update_matches_autograd_update(env, hid, monkeypatch):
    """train() through the hand-written chain at H = 256 and 512 vs manual_update=False, fast_path=False (nn.Linear,
    autograd, clip_grad_norm_, torch.optim.Adam) from the same seed and rollout (collected with the fast path on in
    both runs): parameters within 2e-5 but for at most 1 in 1000 entries (those within 2 lr per Adam step, see below),
    losses within 1e-4 relative.  The plan is the kernel chain ('mlp_chain') on slabs."""
    n, h = 64, 32
    params, losses = {}, {}
    for manual in (True, False):
        plans = []
        vec, pol, data = train_run(env, n, h, hid, manual, monkeypatch, plans)
        clean_pufferl.evaluate(data)              # the same rollout for both: fast_path is switched off for train()
        pol.policy.fast_path = manual
        clean_pufferl.train(data)
        params[manual] = [p.detach().cpu().clone() for p in pol.parameters()]
        losses[manual] = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy,
                                   data.losses.approx_kl, data.losses.clipfrac, data.losses.explained_variance])
        if manual:
            assert (plans[-1].engine, plans[-1].form) == ('mlp_chain', 'slabs'), plans[-1]
            assert data.manual_update.hid == hid and data.manual_update.used_fused is False
        else:
            assert plans[-1].engine == 'model' and data.manual_update is None
        clean_pufferl.close(data)
    # Adam's first steps move an entry by about lr whatever the size of its gradient, so an entry whose minibatch
    # gradient is a cancellation down to fp32 rounding noise may step the other way in one of the two runs: such
    # entries may differ by up to 2 lr per optimizer step.  All others within 2e-5, and at most 1 in 1000 entries past it.
    cfg = make_config(n, h)
    steps = cfg.update_epochs * (n * h // cfg.minibatch_size)
    d = torch.cat([(a - b).abs().reshape(-1) for a, b in zip(params[True], params[False])])
    over = [(name, int(((a - b).abs() > 2e-5).sum()), float((a - b).abs().max()))
            for name, a, b in zip(('W_enc', 'b_enc', 'W_dec', 'b_dec', 'W_val', 'b_val'), params[True], params[False])]
    print(f'[manual-update] {env} H={hid}: param diff {float(d.max()):.2e}; entries past 2e-5 per parameter {over}',
          flush=True)
    assert float(d.max()) <= 2 * cfg.learning_rate * steps, float(d.max())
    assert int((d > 2e-5).sum()) <= d.numel() // 1000, over
    assert np.allclose(losses[True], losses[False], rtol=1e-4, atol=1e-6), (losses[True], losses[False])


@pytest.mark.parametrize('hid', [256, 512])
@pytest.mark.parametrize('env', ['squared', 'breakout'])
def test_manual_update_inside_train_graph(env, hid, monkeypatch):
    """The chain at H > 128 captured whole in the train graph replays to the parameters of eager execution (within
    1e-4); the plan is ('mlp_chain', 'slabs', 'whole').  Breakout at H > 128 runs the per-step rollout loop (its
    persistent rollout kernel is built for H = 128), with the one-kernel policy step captured in the rollout graph."""
    n, h = 128, 32
    out = {}
    for graph in (False, True):
        plans = []
        vec, pol, data = train_run(env, n, h, hid, True, monkeypatch, plans, cuda_graph_train=graph,
                                   cuda_graph_rollout=graph, cuda_graph=graph)
        for _ in range(3):
            clean_pufferl.evaluate(data)
            clean_pufferl.train(data)
        p = plans[-1]
        assert (p.engine, p.form, p.capture) == ('mlp_chain', 'slabs', 'whole' if graph else None), p
        assert (data.train_graph_state == 2) == graph
        assert getattr(data, 'fused_rollouts', 0) == 0
        if env == 'breakout':
            assert not vec.fused_rollout_ok(data.experience, pol)
            assert pol._ticket is not None                 # the rollout ran pb_policy_mlp_sample
            if graph:
                assert data.graph_state == 2
        out[graph] = torch.cat([q.detach().reshape(-1).cpu() for q in pol.parameters()])
        clean_pufferl.close(data)
    assert float((out[True] - out[False]).abs().max()) < 1e-4


def test_password_learns_at_hidden_256():
    """password (tests/test_gpu_ocean_learning.py settings, seed 1, its 20-iteration budget) with Default(hidden_size=256)
    reaches score >= 0.9 through the H = 256 kernels: the fast-path forward and pb_sample_logits at rollout time (its
    observations are narrower than 128 features), the hand-written chain captured in the train graph."""
    from test_gpu_ocean_learning import BUDGET, N, make_config as ocean_config, metric, passed
    torch.manual_seed(1)
    vec = pvec.make(ocean.env_creator('password'), num_envs=N, backend=pvec.B200)
    pol = cleanrl.Policy(models.Default(vec.driver_env, hidden_size=256), fused_sample=True, seed=1).cuda()
    data = clean_pufferl.create(ocean_config(seed=1), vec, pol)
    history = []
    for _ in range(BUDGET['password']):
        clean_pufferl.evaluate(data)
        history.append(metric('password', data))
        if passed('password', history[-1]):
            break
        clean_pufferl.train(data)
        assert data.manual_update is not None and data.manual_update.hid == 256
        assert data.train_minibatch_path == 'slabs' and data.train_graph_state in (1, 2)
    clean_pufferl.close(data)
    print(f'[password, H=256] {len(history)} rollouts; last metrics {history[-3:]}', flush=True)
    assert passed('password', history[-1]), history
