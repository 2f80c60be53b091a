"""LSTMWrapper(Convolutional) -- the reference's Atari LSTM policy (environments/atari/torch.py: Recurrent) -- trained on
bptt segments read in place: conv1 on segment views (pb_conv1_u8_forward_rows / _wgrad_rows, csrc/nature_conv1.cu)
against the dense entry points on a gathered copy, their canaries, determinism, capture and refusals;
LSTMWrapper.forward_segments against forward; train()'s 'cudnn_conv' engine on pong and breakout_pixels against its
eager, gathered and reference-loss ('cudnn') counterparts; C4 at full size.

Reference: clean_pufferl.py:466-482 (minibatch mb holds the bptt segments r*n_mb + mb), :186-244 (the minibatch update,
the LSTM state carried from one minibatch to the next, :188-191)."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from pufferlib_b200 import _native, models

pytestmark = pytest.mark.gpu

ROW = 4 * 84 * 84
Y_ROW = 32 * 400
P = _native.ptr


def lib():
    return _native.lib()


def rollout_frames(envs, groups, steps, nm=2, mb=1, seed=0, outside=255):
    """An arrival-order rollout buffer [H*N, 4, 84, 84] (H = steps * groups * nm, N = envs) of random frames in which
    every frame outside minibatch mb is `outside`, the segment view [E, G, T, 4, 84, 84] of minibatch mb (what
    Experience.segment_obs gives, with the rollout buffer's real strides) and its gathered copy."""
    horizon = steps * groups * nm
    gen = torch.Generator(device='cuda').manual_seed(seed)
    obs = torch.randint(0, 256, (horizon * envs, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=gen)
    window = torch.arange(horizon, device='cuda') // steps
    obs.view(horizon, envs, ROW)[window % nm != mb] = outside
    view = obs.view(groups, nm, steps, envs, 4, 84, 84)[:, mb].permute(2, 0, 1, 3, 4, 5)
    return obs, view, view.contiguous()


def segments(view):
    return view.shape[0] * view.shape[1], view.shape[2], view.shape[1], view.stride(0), view.stride(1), view.stride(2)


def weights(seed):
    torch.manual_seed(seed)
    conv = models.layer_init(torch.nn.Conv2d(4, 32, 8, stride=4)).cuda()
    with torch.no_grad():
        conv.bias.uniform_(-0.1, 0.1)
    return conv.weight.detach().contiguous(), conv.bias.detach().contiguous()


def canaried(n, fill, extra=16):
    buf = torch.full((n + extra,), fill, dtype=torch.float32, device='cuda')
    return buf, buf[:n]


def forward_dense(x, w, b):
    m = x.shape[0]
    yb, y = canaried(m * Y_ROW, -7.0)
    _native.check(lib().pb_conv1_u8_forward(P(x), x.stride(0), m, P(w), P(b), P(y), _native.stream_ptr()))
    assert bool((yb[m * Y_ROW:] == -7.0).all()), 'rows after y were written'
    return y.view(m, 32, 20, 20)


def forward_rows(view, w, b):
    m = view.shape[0] * view.shape[1] * view.shape[2]
    yb, y = canaried(m * Y_ROW, -7.0)
    _native.check(lib().pb_conv1_u8_forward_rows(P(view), *segments(view), P(w), P(b), P(y), _native.stream_ptr()))
    assert bool((yb[m * Y_ROW:] == -7.0).all()), 'rows after y were written'
    return y.view(m, 32, 20, 20)


def wgrad(x, y, dy, rows):
    m = y.shape[0]
    dwb, dw = canaried(32 * 256, float('nan'))
    dbb, db = canaried(32, float('nan'))
    nws = lib().pb_conv1_u8_wgrad_workspace_bytes(m)
    wsb = torch.full((nws + 64,), 0xA5, dtype=torch.uint8, device='cuda')
    if rows:
        _native.check(lib().pb_conv1_u8_wgrad_rows(P(x), *segments(x), P(y), P(dy), P(dw), P(db), P(wsb), nws,
                                                   _native.stream_ptr()))
    else:
        _native.check(lib().pb_conv1_u8_wgrad(P(x), x.stride(0), m, P(y), P(dy), P(dw), P(db), P(wsb), nws,
                                              _native.stream_ptr()))
    assert bool(dwb[32 * 256:].isnan().all()) and bool(dbb[32:].isnan().all()), 'elements after dw / db were written'
    assert bool((wsb[nws:] == 0xA5).all()), 'bytes after the workspace were written'
    return dw.view(32, 256), db


# ---- 1. the C ABI -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('steps', [1, 8, 16])
@pytest.mark.parametrize('groups', [1, 2, 4])
@pytest.mark.parametrize('envs', [1, 3, 37])
def test_rows_bitwise_vs_dense_on_gathered_copy(envs, groups, steps):
    """E envs x G windows = E*G segments of T steps read from the rollout buffer in place: y, dW and db bitwise equal to
    the dense entry points on the gathered copy; the frames outside the view (255) and then the same frames as 0 change
    nothing; canaries after y, dw, db and the workspace intact."""
    w, b = weights(envs * 7 + groups)
    _, view, gathered = rollout_frames(envs, groups, steps, seed=envs + 10 * groups + 100 * steps)
    m = envs * groups * steps
    x = gathered.view(m, 4, 84, 84)
    y_d, y_r = forward_dense(x, w, b), forward_rows(view, w, b)
    assert torch.equal(y_d, y_r)
    dy = torch.randn(m, 32, 20, 20, device='cuda', generator=torch.Generator(device='cuda').manual_seed(m))
    dw_d, db_d = wgrad(x, y_d, dy, rows=False)
    dw_r, db_r = wgrad(view, y_r, dy, rows=True)
    assert torch.equal(dw_d, dw_r) and torch.equal(db_d, db_r)
    _, view0, _ = rollout_frames(envs, groups, steps, seed=envs + 10 * groups + 100 * steps, outside=0)
    assert torch.equal(forward_rows(view0, w, b), y_d)
    dw0, db0 = wgrad(view0, y_r, dy, rows=True)
    assert torch.equal(dw0, dw_d) and torch.equal(db0, db_d)


def test_rows_deterministic_eager_and_graph():
    """2 048 rows (64 envs x 2 windows x 16 steps): two eager calls and two replays of a captured graph agree bitwise."""
    w, b = weights(1)
    _, view, _ = rollout_frames(64, 2, 16, seed=1)
    m = 64 * 2 * 16
    y1, y2 = forward_rows(view, w, b), forward_rows(view, w, b)
    assert torch.equal(y1, y2)
    dy = torch.randn(m, 32, 20, 20, device='cuda')
    (a1, c1), (a2, c2) = wgrad(view, y1, dy, rows=True), wgrad(view, y1, dy, rows=True)
    assert torch.equal(a1, a2) and torch.equal(c1, c2)
    yg, dwg, dbg = torch.empty_like(y1), torch.empty(32, 256, device='cuda'), torch.empty(32, device='cuda')
    ws = torch.empty(lib().pb_conv1_u8_wgrad_workspace_bytes(m), dtype=torch.uint8, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            sp = _native.stream_ptr(s)
            _native.check(lib().pb_conv1_u8_forward_rows(P(view), *segments(view), P(w), P(b), P(yg), sp))
            _native.check(lib().pb_conv1_u8_wgrad_rows(P(view), *segments(view), P(yg), P(dy), P(dwg), P(dbg), P(ws),
                                                       ws.numel(), sp))
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        yg.zero_(), dwg.zero_(), dbg.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(yg, y1) and torch.equal(dwg, a1) and torch.equal(dbg, c1)


def test_rows_refusals_launch_nothing():
    """PB_ERR_INVALID before any launch for batch < 0, steps < 1, groups < 1, batch % groups != 0, a stride below a row
    or not a multiple of 16, null or misaligned pointers and a short workspace; batch = 0 is PB_OK without a launch."""
    L = lib()
    _, view, _ = rollout_frames(4, 2, 4, seed=0)
    m = 32
    w, b = weights(0)
    y = torch.empty(m, 32, 20, 20, device='cuda')
    dw, db = torch.empty(32, 256, device='cuda'), torch.empty(32, device='cuda')
    nws = L.pb_conv1_u8_wgrad_workspace_bytes(m)
    ws = torch.empty(nws + 16, dtype=torch.uint8, device='cuda')
    sp = _native.stream_ptr()
    off = lambda t_, k: C.c_void_p(t_.data_ptr() + k)  # noqa: E731
    good = dict(x=P(view), batch=8, steps=4, groups=2, se=view.stride(0), sg=view.stride(1), st=view.stride(2))
    bad_geom = [dict(x=None), dict(x=off(view, 8)), dict(batch=-2), dict(steps=0), dict(steps=-1), dict(groups=0),
                dict(groups=-2), dict(groups=3), dict(batch=9)]
    for k in ('se', 'sg', 'st'):
        bad_geom += [{k: ROW - 16}, {k: ROW + 8}, {k: 0}, {k: -ROW}]
    before = L.pb_launch_count()
    for bad in bad_geom:
        a = dict(good, **bad)
        geom = (a['x'], a['batch'], a['steps'], a['groups'], a['se'], a['sg'], a['st'])
        assert L.pb_conv1_u8_forward_rows(*geom, P(w), P(b), P(y), sp) == _native.PB_ERR_INVALID, bad
        assert L.pb_conv1_u8_wgrad_rows(*geom, P(y), P(y), P(dw), P(db), P(ws), nws, sp) == _native.PB_ERR_INVALID, bad
    geom = tuple(good.values())
    for fw in [(None, P(b), P(y)), (off(w, 4), P(b), P(y)), (P(w), None, P(y)), (P(w), off(b, 2), P(y)),
               (P(w), P(b), None), (P(w), P(b), off(y, 4))]:
        assert L.pb_conv1_u8_forward_rows(*geom, *fw, sp) == _native.PB_ERR_INVALID, fw
    for wg in [(off(y, 4), P(y), P(dw), P(db), P(ws), nws), (P(y), None, P(dw), P(db), P(ws), nws),
               (P(y), P(y), None, P(db), P(ws), nws), (P(y), P(y), off(dw, 2), P(db), P(ws), nws),
               (P(y), P(y), P(dw), None, P(ws), nws), (P(y), P(y), P(dw), P(db), None, nws),
               (P(y), P(y), P(dw), P(db), off(ws, 4), nws), (P(y), P(y), P(dw), P(db), P(ws), nws - 4)]:
        assert L.pb_conv1_u8_wgrad_rows(*geom, *wg, sp) == _native.PB_ERR_INVALID, wg
    assert 'pb_conv1_u8_wgrad_rows' in _native.last_error()
    zero = (P(view), 0, 4, 2, view.stride(0), view.stride(1), view.stride(2))
    assert L.pb_conv1_u8_forward_rows(*zero, P(w), P(b), P(y), sp) == _native.PB_OK
    assert L.pb_conv1_u8_wgrad_rows(*zero, P(y), P(y), P(dw), P(db), P(ws), 16, sp) == _native.PB_OK
    assert L.pb_launch_count() == before


# ---- 2. the model -----------------------------------------------------------------------------------------------------
def pong_env():
    from test_gpu_policy_lstm import fake_env
    return fake_env((4, 84, 84), 6, np.uint8)


def conv_lstm(seed):
    torch.manual_seed(seed)
    env = pong_env()
    return models.LSTMWrapper(env, models.Convolutional(env), input_size=512, hidden_size=512).cuda()


def test_forward_segments_bitwise_vs_forward_on_gathered_copy(monkeypatch):
    """forward_segments on the segment view (16 envs x 2 windows x 8 steps) equals forward on the gathered copy
    [32, 8, 4, 84, 84] bit for bit: logits, values, the final state and every parameter's gradient of a loss on the
    outputs (cuDNN in its deterministic mode, as train() runs it with torch_deterministic).  conv1 runs on the rows
    entry points, and no copy of the frames is made."""
    monkeypatch.setattr(torch.backends.cudnn, 'deterministic', True)
    a, b_ = conv_lstm(3), conv_lstm(3)
    envs, groups, steps = 16, 2, 8
    _, view, gathered = rollout_frames(envs, groups, steps, seed=5)
    bsz = envs * groups
    gen = torch.Generator(device='cuda').manual_seed(1)
    state = tuple(torch.randn(1, bsz, 512, device='cuda', generator=gen) * 0.5 for _ in range(2))
    ra, rb = torch.randn(bsz * steps, 6, device='cuda', generator=gen), torch.randn(bsz * steps, 1, device='cuda', generator=gen)
    seen = []
    orig = models._Conv1U8Function.apply
    monkeypatch.setattr(models._Conv1U8Function, 'apply',
                        lambda x, *r: seen.append((x.dim(), x.data_ptr(), x.stride())) or orig(x, *r))
    ls, vs, (hs, cs) = a.forward_segments(view, state)
    lg, vg, (hg, cg) = b_(gathered.view(bsz, steps, 4, 84, 84), state)
    assert seen[0] == (6, view.data_ptr(), view.stride()), 'conv1 did not read the view in place'
    assert [d for d, _, _ in seen] == [6, 4]
    assert torch.equal(ls, lg) and torch.equal(vs, vg) and torch.equal(hs, hg) and torch.equal(cs, cg)
    ((ls * ra).sum() + (vs * rb).sum()).backward()
    ((lg * ra).sum() + (vg * rb).sum()).backward()
    for (name, pa), pb in zip(a.named_parameters(), b_.parameters()):
        assert torch.equal(pa.grad, pb.grad), name


def test_forward_segments_declines_what_conv1_cannot_read():
    """None (train() keeps today's path) for a view on the CPU, with a misaligned stride, float frames, or an inner
    policy without encode_segments."""
    net = conv_lstm(0)
    _, view, _ = rollout_frames(2, 1, 4, seed=0)
    assert net.forward_segments(view.cpu(), None) is None
    assert net.forward_segments(view.float(), None) is None
    odd = torch.zeros(2 * ROW + 8, dtype=torch.uint8, device='cuda')
    assert net.forward_segments(torch.as_strided(odd, (2, 1, 1, 4, 84, 84), (ROW + 8, ROW, ROW, 7056, 84, 1)), None) is None
    from test_gpu_policy_lstm import fake_env
    env = fake_env((49,), 4)
    assert models.LSTMWrapper(env, models.Default(env)).cuda().forward_segments(torch.rand(2, 1, 4, 49).cuda(), None) is None


# ---- 3. through the trainer -------------------------------------------------------------------------------------------
def trainer(kind, n, h, bptt, nm, lr, **kw):
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    from test_gpu_config_updates import ppo_config
    vec = pvec.make(ocean.env_creator(kind), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    net = models.LSTMWrapper(vec.driver_env, models.Convolutional(vec.driver_env), input_size=512, hidden_size=512)
    pol = cleanrl.RecurrentPolicy(net, seed=3).cuda()
    cfg = dict(fused_loss=True, learning_rate=lr, cuda_graph=True)
    cfg.update(kw)
    return clean_pufferl.create(ppo_config(kind, n, h, bptt, nm, **cfg), vec, pol)


def loss_vector(data):
    return np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy, data.losses.approx_kl,
                     data.losses.clipfrac, data.losses.explained_variance])


@pytest.mark.parametrize('kind', ['pong', 'breakout_pixels'])
def test_train_plan_capture_and_paths(kind, monkeypatch):
    """train() on `kind` (256 envs x 32 steps, bptt 8, 2 minibatches, 2 epochs), evaluate() + train() twice per trainer,
    every trainer from the same seeds:
      captured  plan ('cudnn_conv', 'segments', 'whole'), train graph state 2 after the second call, b_obs never allocated;
      eager     cuda_graph_train=False: bitwise the captured trainer's parameters and losses after both calls;
      gathered  zero_copy_minibatches=False: plan ('cudnn_conv', 'gathered'), bitwise the eager trainer;
      reference fused_loss=False (today's path, plan ('cudnn', 'gathered', None)): from the same first rollout, losses
                within 2e-3 relative and per parameter tensor a median difference of at most lr / 10 and a maximum of
                at most 8 lr (each of the 4 Adam steps moves an element by about lr at most in each trainer), as
                test_gpu_nature_trunk.test_pong_train_vs_refused derives them.
    The rollouts of the first iteration are the same in all four (the rollout is unchanged)."""
    from pufferlib_b200 import clean_pufferl
    n, h, bptt, nm, lr = 256, 32, 8, 2, 2.5e-4
    plans = []
    update_plan = clean_pufferl.update_plan
    monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(update_plan(d)) or plans[-1])
    variants = {'captured': {}, 'eager': dict(cuda_graph_train=False),
                'gathered': dict(cuda_graph_train=False, zero_copy_minibatches=False), 'reference': dict(fused_loss=False)}
    expect = {'captured': ('cudnn_conv', 'segments', 'whole'), 'eager': ('cudnn_conv', 'segments', None),
              'gathered': ('cudnn_conv', 'gathered', None), 'reference': ('cudnn', 'gathered', None)}
    res = {}
    for name, kw in variants.items():
        data = trainer(kind, n, h, bptt, nm, lr, **kw)
        out = []
        for it in range(2):
            clean_pufferl.evaluate(data)
            roll = data.experience.obs.clone() if it == 0 else None
            clean_pufferl.train(data)
            p = plans[-1]
            assert (p.engine, p.form, p.capture) == expect[name], (name, p)
            assert np.isfinite(loss_vector(data)[:5]).all(), name
            params = {k: q.detach().clone() for k, q in data.policy.named_parameters()}
            out.append((roll, params, loss_vector(data)))
        if name == 'captured':
            assert data.train_graph_state == 2, data.msg
            print(f'{kind}: rollout graph state {data.graph_state}, train graph state {data.train_graph_state}, '
                  f'train graph launches {data.train_graph_launches}', flush=True)
        if name != 'reference' and expect[name][1] == 'segments':
            assert data.experience._b_obs is None, 'b_obs was allocated on the segments plan'
        res[name] = out
        clean_pufferl.close(data)
    for name in ('eager', 'gathered', 'reference'):
        assert torch.equal(res[name][0][0], res['captured'][0][0]), f'{name}: first rollout differs'
    for a_, b_ in (('captured', 'eager'), ('eager', 'gathered')):
        for it in range(2):
            assert np.array_equal(res[a_][it][2], res[b_][it][2], equal_nan=True), (a_, b_, it)
            for k, v in res[a_][it][1].items():
                assert torch.equal(v, res[b_][it][1][k]), (a_, b_, it, k)
    new, ref = res['eager'][0], res['reference'][0]
    print(f'{kind} losses cudnn_conv {new[2]} reference {ref[2]}', flush=True)
    assert np.allclose(new[2], ref[2], rtol=2e-3, atol=1e-5)
    for k, v in new[1].items():
        d = (v - ref[1][k]).abs().double().flatten()
        print(f'{k:32s} {d.numel():8d} elements: max {float(d.max()):.2e} median {float(d.median()):.2e}', flush=True)
        assert float(d.median()) <= lr / 10, k
        assert float(d.max()) <= 8 * lr, k


# ---- 4. full size -----------------------------------------------------------------------------------------------------
def c4_lstm_budget(n, h, mb):
    """Peak device memory allowed for C4 with LSTMWrapper(Convolutional) on the segments plan: the rollout observations
    once (n * h rows of 28 224 bytes; no b_obs), per minibatch row conv1's saved y1 and its gradient (2 * 12 800 floats),
    the other layers' saved activations and gradients (3 * (5184 + 3136 + 512) floats: conv2, conv3, the Linear), the
    LSTM's input, output, their gradients and cuDNN's reserve (12 * 512 floats), plus 4 GiB for the per-row rollout
    tensors, parameters, optimizer state, cuDNN workspaces and the allocator."""
    acts = mb * 4 * (2 * Y_ROW + 3 * (5184 + 3136 + 512) + 12 * 512)
    return n * h * ROW + acts + 4 * 2 ** 30


def test_pong_c4_full_size_trains_twice():
    """pong at 4 096 envs x 128 steps, bptt 16, 4 minibatches of 131 072 rows, cuda_graph=True: two evaluate() + train()
    iterations with finite losses on the 'cudnn_conv' segments plan, both graph states reported, peak memory under
    c4_lstm_budget."""
    from pufferlib_b200 import clean_pufferl
    n, h, nm = 4096, 128, 4
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    data = trainer('pong', n, h, 16, nm, 2.5e-4)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        assert np.isfinite(loss_vector(data)[:5]).all()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    budget = c4_lstm_budget(n, h, n * h // nm)
    print(f'pong C4 LSTM(Conv): peak {peak / 2 ** 30:.2f} GiB, budget {budget / 2 ** 30:.2f} GiB, path '
          f'{data.train_minibatch_path}, rollout graph state {data.graph_state}, train graph state '
          f'{data.train_graph_state} ({data.msg})', flush=True)
    assert data.train_minibatch_path == 'segments' and data.experience._b_obs is None
    assert peak <= budget
    clean_pufferl.close(data)
