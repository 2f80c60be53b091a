"""The recurrent PPO update read in place and captured: the segment-view entry points pb_lstm_bptt_forward_rows /
pb_lstm_bptt_backward_rows (csrc/lstm_bptt.cu), LSTMWrapper.forward_packed_seq on Experience.segment_obs views
(train_minibatch_path 'segments'), and train() captured in one CUDA graph for RecurrentPolicy(fused_update=True).

Reference: clean_pufferl.py:466-482 (minibatch mb holds the bptt segments r*n_mb + mb), :186-244 (the minibatch update,
the state carried from one minibatch to the next, :188-191)."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from test_gpu_lstm_bptt import forward_kernel, make_net, snapshot_train
from test_gpu_policy_lstm import make_config, sharpen

gpu = pytest.mark.gpu
P = _native.ptr
NAN = float('nan')
LOSSES = ('policy_loss', 'value_loss', 'entropy', 'old_approx_kl', 'approx_kl', 'clipfrac')


def losses(data):
    return {k: float(getattr(data.losses, k)) for k in LOSSES}


@pytest.fixture
def fp32_matmul():
    """Library GEMMs in full fp32 for the test's duration.  Under TF32 ('high', what clean_pufferl sets) the library may
    run one of two GEMM shapes on tensor cores and the other in fp32, which differ by TF32 rounding (~5e-4), not by
    summation order; the comparisons that use this fixture are about summation order."""
    prev = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision('highest')
    yield
    torch.set_float32_matmul_precision(prev)


def test_rows_entry_points_refuse_bad_arguments_before_any_launch():
    """PB_ERR_INVALID for groups < 1, batch % groups != 0, strides below a row, null and misaligned pointers;
    PB_ERR_UNSUPPORTED for shapes outside the model envelope; PB_OK without a launch for batch = 0.  No device needed: every
    check comes before any CUDA call (each call below has at least one bad argument, or batch = 0)."""
    lib = _native.lib()
    p, odd8, odd16 = C.c_void_p(256), C.c_void_p(260), C.c_void_p(264)

    def fwd(feats=49, batch=8, steps=16, groups=2, se=49, sg=49 * 64, st=49 * 4, size=128, n_act=8, obs=p, w_enc=p,
            out=p, h0=None, saved=p):
        return lib.pb_lstm_bptt_forward_rows(obs, feats, batch, steps, groups, se, sg, st, h0, None, w_enc, p, p, p, p, p,
                                             size, 128, n_act, out, p, p, saved, None)

    def bwd(batch=8, steps=16, groups=2, de=128, dg=128 * 64, dt=128 * 4, size=128, n_act=8, w_t=p, dz=p, dpre=p,
            c0=None):
        return lib.pb_lstm_bptt_backward_rows(p, p, c0, w_t, p, batch, steps, size, 128, n_act, groups, de, dg, dt, dz,
                                              dpre, None)
    invalid = [fwd(groups=0), fwd(groups=-2), fwd(batch=9), fwd(batch=-2), fwd(steps=0), fwd(se=48), fwd(sg=48),
               fwd(st=48), fwd(se=-49), fwd(obs=None), fwd(out=None), fwd(saved=None), fwd(out=odd8), fwd(h0=odd8),
               fwd(w_enc=odd16),
               bwd(groups=0), bwd(batch=9), bwd(steps=0), bwd(de=127), bwd(dg=126), bwd(dt=0), bwd(de=129),
               bwd(dt=130 + 1), bwd(dz=None), bwd(dpre=None), bwd(dpre=odd8), bwd(c0=odd8), bwd(w_t=odd16)]
    assert all(rc == _native.PB_ERR_INVALID for rc in invalid), invalid
    assert 'pb_lstm_bptt_backward_rows' in _native.last_error()
    unsupported = [fwd(feats=129), fwd(feats=0), fwd(size=64), fwd(n_act=16), fwd(n_act=0), bwd(size=64), bwd(n_act=16)]
    assert all(rc == _native.PB_ERR_UNSUPPORTED for rc in unsupported), unsupported
    assert fwd(batch=0) == bwd(batch=0) == _native.PB_OK
    assert fwd(batch=0, groups=4, obs=None) == bwd(batch=0, groups=4, dpre=None) == _native.PB_OK     # nothing to do


def test_forward_packed_seq_declines_segment_views_it_cannot_read_on_cpu():
    """forward_packed_seq returns None (the caller keeps the cuDNN path) for [E, G, T, *obs] views on the CPU or with the
    wrong observation shape."""
    torch.manual_seed(0)
    from test_gpu_policy_lstm import fake_env
    env = fake_env((49,), 4)
    net = models.LSTMWrapper(env, models.Default(env), input_size=128, hidden_size=128)
    assert net.forward_packed_seq(torch.rand(5, 2, 8, 49), None) is None        # not CUDA
    assert net.forward_packed_seq(torch.rand(5, 2, 8, 7, 7), None) is None      # wrong observation shape


def segment_setup(groups, steps, feats, nm=3, mb=1, envs=150, seed=0):
    """Arrival-order observations [H*N, F] (H = steps * groups * nm) in which every row outside minibatch mb is NaN, the
    segment view [E, G, T, F] of minibatch mb, and pb_minibatch_gather's copy [B, T, F] of the same minibatch."""
    horizon, n = steps * groups * nm, envs
    gen = torch.Generator(device='cuda').manual_seed(seed)
    obs = torch.rand(horizon * n, feats, device='cuda', generator=gen) * 2 - 1
    window = torch.arange(horizon, device='cuda') // steps
    obs.view(horizon, n, feats)[window % nm != mb] = NAN
    seg = obs.view(groups, nm, steps, n, feats)[:, mb].permute(2, 0, 1, 3)
    bsz = n * groups
    gathered = torch.full((bsz, steps, feats), NAN, device='cuda')
    _native.check(_native.lib().pb_minibatch_gather(P(obs), P(gathered), 4 * feats, n, horizon, nm, bsz, steps, mb, 1,
                                                    _native.stream_ptr()))
    return obs, seg, gathered


def forward_rows_kernel(net, seg, h0=None, c0=None, guard=5):
    """pb_lstm_bptt_forward_rows on the segment view [E, G, T, F], NaN canaries past every output."""
    e_, g_, steps, feats = seg.shape
    bsz, m = e_ * g_, e_ * g_ * steps
    n_act = net.policy.decoder.weight.shape[0]
    with torch.no_grad():
        w_enc, b_enc, w_gates, b_gates, w_cat, b_cat = net.fused_operands()
    out = torch.full((m + guard, w_cat.shape[0]), NAN, device='cuda')
    hT, cT = torch.full((bsz + guard, 128), NAN, device='cuda'), torch.full((bsz + guard, 128), NAN, device='cuda')
    saved = torch.full((m + guard, 1024), NAN, device='cuda')
    _native.check(_native.lib().pb_lstm_bptt_forward_rows(
        P(seg), feats, bsz, steps, g_, seg.stride(0), seg.stride(1), seg.stride(2), P(h0), P(c0), P(w_enc), P(b_enc),
        P(w_gates), P(b_gates), P(w_cat), P(b_cat), 128, 128, n_act, P(out), P(hT), P(cT), P(saved),
        _native.stream_ptr()))
    torch.cuda.synchronize()
    for buf, n in ((out, m), (hT, bsz), (cT, bsz), (saved, m)):
        assert bool(buf[n:].isnan().all()), 'a row past the end was written'
    return out[:m], hT[:bsz], cT[:bsz], saved[:m]


def backward_kernel(net, dout, saved, c0, bsz, steps, groups=None, envs=None, guard=5):
    """pb_lstm_bptt_backward (groups None) or pb_lstm_bptt_backward_rows with the segment view's dPre strides ->
    (dz, dpre), NaN canaries past both."""
    m, n_act = bsz * steps, net.policy.decoder.weight.shape[0]
    dz, dpre = torch.full((m + guard, 512), NAN, device='cuda'), torch.full((m + guard, 128), NAN, device='cuda')
    w_cat = net.fused_operands()[4]
    lib = _native.lib()
    if groups is None:
        _native.check(lib.pb_lstm_bptt_backward(
            P(dout), P(saved), P(c0), P(net.gate_weights_transposed()), P(w_cat), bsz, steps, 128, 128, n_act, P(dz),
            P(dpre), _native.stream_ptr()))
    else:
        _native.check(lib.pb_lstm_bptt_backward_rows(
            P(dout), P(saved), P(c0), P(net.gate_weights_transposed()), P(w_cat), bsz, steps, 128, 128, n_act, groups,
            128, 128 * steps * envs, 128 * envs, P(dz), P(dpre), _native.stream_ptr()))
    torch.cuda.synchronize()
    assert bool(dz[m:].isnan().all()) and bool(dpre[m:].isnan().all()), 'a row past the end was written'
    return dz[:m], dpre[:m]


@gpu
@pytest.mark.parametrize('init', [False, True])
@pytest.mark.parametrize('n_act', [4, 8, 15])
@pytest.mark.parametrize('feats', [1, 49, 128])
@pytest.mark.parametrize('steps', [1, 16])
@pytest.mark.parametrize('groups', [1, 2, 4])
def test_segment_view_matches_gathered_minibatch(groups, steps, feats, n_act, init, fp32_matmul):
    """The _rows entry points on the segment view of minibatch 1 of 3 (every other row of the rollout buffer is NaN;
    E = 150 envs, so E*G = 150 / 300 / 600 segments leave the last CTA ragged) vs the dense entry points on
    pb_minibatch_gather's copy: the view holds the gathered segments; out, h_T, c_T, the saved rows and dz are bitwise
    equal, dPre is bitwise equal after its row permutation, no NaN reaches an output and no row past an output is
    written; dW_enc from the slab GEMM agrees with the gathered GEMM to summation order (1e-5 of its largest entry,
    both in fp32)."""
    net = make_net(feats, n_act)
    envs = 150
    _, seg, gathered = segment_setup(groups, steps, feats, envs=envs, seed=31 * groups + steps + feats + n_act)
    bsz, m = envs * groups, envs * groups * steps
    assert torch.equal(seg.reshape(bsz, steps, feats), gathered)        # segment r = e*G + g is the reference's row r
    gen = torch.Generator(device='cuda').manual_seed(7 + n_act)
    h0 = (torch.randn(bsz, 128, device='cuda', generator=gen) * 0.5) if init else None
    c0 = torch.randn(bsz, 128, device='cuda', generator=gen) if init else None

    ref = forward_kernel(net, gathered, h0, c0)
    got = forward_rows_kernel(net, seg, h0, c0)
    for name, a, b in zip(('out', 'h_T', 'c_T', 'saved'), got, ref):
        assert bool(a.isfinite().all()), name
        assert torch.equal(a, b), name

    dout = torch.randn(m, ref[0].shape[1], device='cuda', generator=gen) / m ** 0.5
    dout[:, n_act + 1:] = 0
    dz_ref, dpre_ref = backward_kernel(net, dout, ref[3], c0, bsz, steps)
    dz, dpre = backward_kernel(net, dout, got[3], c0, bsz, steps, groups, envs)
    assert bool(dz.isfinite().all()) and bool(dpre.isfinite().all())
    assert torch.equal(dz, dz_ref)
    # dPre row ((b % G) T + t) N + b / G of the segment layout = row b*T + t of the dense one
    assert torch.equal(dpre.view(groups, steps, envs, 128).permute(2, 0, 1, 3).reshape(m, 128), dpre_ref)

    dw_slab = models._gemm_tn(dpre, seg.permute(1, 2, 0, 3).view(groups, steps * envs, feats))
    dw_ref = models._gemm_tn(dpre_ref, gathered.reshape(m, feats))
    err = float((dw_slab - dw_ref).abs().max()) / (float(dw_ref.abs().max()) + 1e-30)
    assert err <= 1e-5, err


def make_recurrent(env, n, fused_update=True, hidden=128, layers=1, seed=3):
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env, hidden_size=hidden), input_size=hidden,
                             hidden_size=hidden, num_layers=layers)
    if hidden == 128 and layers == 1:
        sharpen(net)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=seed, fused_update=fused_update).cuda()
    return vec, net, pol


@gpu
@pytest.mark.parametrize('env,n,h,bptt', [('breakout', 256, 64, 16), ('squared', 64, 32, 8)])
def test_train_zero_copy_segments_match_gathered_minibatches(env, n, h, bptt, monkeypatch, fp32_matmul):
    """train() with the fused BPTT update reading Experience.segment_obs views (zero_copy_minibatches=True) vs the
    gathered b_obs copy (False), from one parameter snapshot and one stored rollout, two minibatches of G = 2 time
    windows, two epochs.  The segment run allocates no b_obs; the state handed to the second minibatch and the first
    step's gradients are bitwise equal, except dW_enc and db_enc (the sums over dPre's rows run in slab order: within 1e-5
    of the largest entry); with the snapshot parameters the whole per-minibatch carry (out, h, c of every minibatch) is
    bitwise equal; the parameters after train() agree to 2e-5 and the losses to summation order.  The weight-gradient
    GEMMs run in fp32 here (fp32_matmul) so that dW_enc differs by summation order only."""
    vec, net, pol = make_recurrent(env, n)
    data = clean_pufferl.create(make_config(n, h, env=env, bptt_horizon=bptt, update_epochs=2), vec, pol)
    clean_pufferl.evaluate(data)
    params0 = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    opt0 = data.optimizer.state_dict()
    res, paths = {}, {}
    for zc in (True, False):                     # segments first: nothing may have allocated b_obs yet
        pol.load_state_dict(params0)
        data.optimizer.load_state_dict(opt0)
        net.invalidate_cache()
        data.config.zero_copy_minibatches = zc
        res[zc] = snapshot_train(data, pol, net, True, monkeypatch)
        paths[zc] = data.train_minibatch_path
        if zc:
            assert data.experience._b_obs is None
    assert paths == {True: 'segments', False: 'gathered'}, paths
    (ra, la, pa, path_a), (rb, lb, pb, path_b) = res[True], res[False]
    assert path_a == path_b == 'fused'
    nm = data.experience.num_minibatches
    assert len(ra['states']) == len(rb['states']) == 2 * nm and ra['states'][0] is None and ra['states'][nm] is None
    for a, b in zip(ra['states'][1], rb['states'][1]):
        assert torch.equal(a, b)
    summed = ('encoder.weight', 'encoder.bias')
    errs = {}
    for k, g in rb['grads'].items():
        if k.endswith(summed):
            errs[k] = float((ra['grads'][k] - g).abs().max()) / float(g.abs().max())
        else:
            assert torch.equal(ra['grads'][k], g), k
    perr = float((pa - pb).abs().max())
    print(f'[segments] {env} n={n} h={h} bptt={bptt}: encoder grad err / max {errs}, param err {perr:.2e}, '
          f'losses {la} vs {lb}', flush=True)
    assert len(errs) == 2 and all(e <= 1e-5 for e in errs.values()), errs
    assert perr <= 2e-5, perr
    for k in la:        # clipfrac: one row crossing the clip edge moves it by 1 / (rows * n_mb)
        assert np.isclose(la[k], lb[k], rtol=1e-4, atol=1e-4), (k, la[k], lb[k])

    # the carry with frozen (snapshot) parameters: every minibatch's output and final state, bitwise
    pol.load_state_dict(params0)
    net.invalidate_cache()
    exp = data.experience
    sa = sb = None
    with torch.no_grad():
        for mb in range(nm):
            oa, _, sa = net.forward_packed_seq(exp.segment_obs(mb), sa)
            ob, _, sb = net.forward_packed_seq(exp.b_obs[mb], sb)
            assert torch.equal(oa, ob) and torch.equal(sa[0], sb[0]) and torch.equal(sa[1], sb[1]), mb
    clean_pufferl.close(data)


def adam_state(opt):
    return [t for p in opt.param_groups[0]['params'] for t in (opt.state[p]['exp_avg'], opt.state[p]['exp_avg_sq'],
                                                                 opt.state[p]['step'])]


@gpu
@pytest.mark.parametrize('env,n,h,bptt', [('breakout', 256, 64, 16), ('squared', 64, 32, 8)])
def test_captured_train_matches_eager_train(env, n, h, bptt):
    """A replay of the captured recurrent update vs an eager train() from the same parameters, Adam state (restored in
    place: the graph holds those tensors) and stored rollout.  The capture ran the fused path on segment views, holds at
    least the 2 * update_epochs * n_mb BPTT launches, and the replay launches nothing from Python; parameters and Adam
    moments agree to 2e-6 (the GAE look-back composes tile aggregates in a timing-dependent order, ~1e-7 run to run), the
    losses closely."""
    vec, net, pol = make_recurrent(env, n)
    cfg = make_config(n, h, env=env, bptt_horizon=bptt, update_epochs=2, cuda_graph=True)
    data = clean_pufferl.create(cfg, vec, pol)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
    assert data.train_graph_state == 2, data.msg
    assert data.train_recurrent_path == 'fused' and data.train_minibatch_path == 'segments'
    nm = data.experience.num_minibatches
    assert data.train_graph_launches >= 2 * cfg.update_epochs * nm, data.train_graph_launches
    clean_pufferl.evaluate(data)
    opt = data.optimizer
    params = list(pol.parameters())
    snap_p = [p.detach().clone() for p in params]
    snap_s = [t.clone() for t in adam_state(opt)]
    replays0, launches0 = data.train_graph_replays, _native.lib().pb_launch_count()
    clean_pufferl.train(data)
    assert data.train_graph_replays == replays0 + 1 and _native.lib().pb_launch_count() == launches0
    got = ([p.detach().clone() for p in params], [t.clone() for t in adam_state(opt)], losses(data))
    with torch.no_grad():
        for p, s in zip(params, snap_p):
            p.copy_(s)
        for t, s in zip(adam_state(opt), snap_s):
            t.copy_(s)
    net.invalidate_cache()
    data.config.cuda_graph_train = False
    clean_pufferl.train(data)
    assert data.train_recurrent_path == 'fused' and data.train_minibatch_path == 'segments'
    ref = ([p.detach() for p in params], adam_state(opt), losses(data))
    perr = max(float((a - b).abs().max()) for a, b in zip(got[0], ref[0]))
    serr = max(float((a.float() - b.float()).abs().max()) for a, b in zip(got[1], ref[1]))
    print(f'[train-graph] {env} n={n} h={h}: param err {perr:.2e}, adam state err {serr:.2e}, losses {got[2]} vs '
          f'{ref[2]}', flush=True)
    assert perr <= 2e-6 and serr <= 2e-6, (perr, serr)
    for k, v in ref[2].items():
        assert np.isclose(got[2][k], v, rtol=1e-4, atol=1e-4), (k, got[2][k], v)
    clean_pufferl.close(data)


@gpu
def test_graphed_recurrent_training_matches_eager_training():
    """The three-iteration loop of test_gpu_experience.py::test_graphed_training_matches_eager_training with
    RecurrentPolicy(fused_sample=True, fused_update=True): rollout and train graphs on vs off, anneal_lr, same config
    (so the same capturable Adam) and the same assertions."""
    n, h = 64, 32
    params, rollouts = {}, {}
    for mode in ('eager', 'graph'):
        vec, net, pol = make_recurrent('breakout', n, seed=7)
        g = mode == 'graph'
        data = clean_pufferl.create(make_config(n, h, env='breakout', cuda_graph=True, cuda_graph_rollout=g,
                                                cuda_graph_train=g, anneal_lr=True, total_timesteps=20 * n * h), vec, pol)
        rollouts[mode], params[mode] = [], []
        for it in range(3):
            clean_pufferl.evaluate(data)
            rollouts[mode].append(data.experience.actions.cpu().numpy().copy())
            clean_pufferl.train(data)
            assert data.train_recurrent_path == 'fused'
            params[mode].append([p.detach().cpu().clone() for p in pol.parameters()])
        if g:
            assert data.train_graph_state == 2 and data.train_graph_replays == 2 and data.graph_replays == 2, data.msg
        else:
            assert data.train_graph_state != 2 and data.graph_replays == 0
        clean_pufferl.close(data)
    agree = [float((a == b).mean()) for a, b in zip(rollouts['eager'], rollouts['graph'])]
    diffs = [max(float((a - b).abs().max()) for a, b in zip(pa, pb)) for pa, pb in zip(params['eager'], params['graph'])]
    print(f'[train-graph-loop] action agreement {agree}, parameter diffs {diffs}', flush=True)
    assert agree[0] == 1.0 and agree[1] > 0.9995 and agree[2] > 0.98, (agree, diffs)
    assert diffs[0] <= 2e-6 and diffs[1] <= 2e-5, (agree, diffs)


@gpu
@pytest.mark.parametrize('kind', ['hidden64', 'two_layers', 'uint8_obs', 'fast_path_off', 'fused_update_off'])
def test_uncovered_recurrent_updates_stay_eager(kind):
    """With cuda_graph=True a recurrent update that does not run on the BPTT kernels is never captured: two train() calls
    (the second is where a capture would happen) run the cuDNN path eagerly and compute bit-identically what the same two
    calls compute with cuda_graph=False, from the same snapshot and rollout."""
    env = 'snake' if kind == 'uint8_obs' else 'squared'
    hidden, layers = (64 if kind == 'hidden64' else 128), (2 if kind == 'two_layers' else 1)
    n, h = 64, 16
    vec, net, pol = make_recurrent(env, n, fused_update=kind != 'fused_update_off', hidden=hidden, layers=layers)
    if kind == 'fast_path_off':
        net.policy.fast_path = False
    data = clean_pufferl.create(make_config(n, h, env=env, bptt_horizon=8, update_epochs=1, cuda_graph=True), vec, pol)
    clean_pufferl.evaluate(data)
    params0 = {k: v.detach().clone() for k, v in pol.state_dict().items()}
    opt0 = data.optimizer.state_dict()
    res = {}
    for graph in (True, False):
        pol.load_state_dict(params0)
        data.optimizer.load_state_dict(opt0)
        net.invalidate_cache()
        data.config.cuda_graph = graph
        runs = []
        for _ in range(2):
            clean_pufferl.train(data)
            assert data.train_graph_state != 2 and data.train_recurrent_path == 'cudnn', (kind, data.train_graph_state)
            assert data.train_minibatch_path == 'gathered'
            runs.append((torch.cat([p.detach().reshape(-1) for p in pol.parameters()]).clone(), losses(data)))
        res[graph] = runs
    for (pa, la), (pb, lb) in zip(res[True], res[False]):
        assert torch.equal(pa, pb) and la == lb
    clean_pufferl.close(data)
