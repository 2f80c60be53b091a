"""One-frame observations for the pixel kinds (`framestack=1`: rows of (1, 84, 84), 7 056 bytes) and NatureCNN's conv1 on
them (csrc/nature_conv1.cu at C = 1):
  1. the env against the one-frame oracle (tests/framestack_oracle.py), bit for bit, plain and with the reference's
     preprocessing stack, at sizes up to one where every CTA's ring wraps, and in every vectoriser mode;
  2. the env against itself: S = 1 is the newest frame of S = 4 from the same seed and actions;
  3. a captured rollout, and the refusals;
  4. conv1's _ex kernels at C = 1: exact and fp64 checks, segment views, determinism, capture, and _ex at C = 4 being
     the existing entry points;
  5. Convolutional(framestack=1) on the fast path, and train() with it (plain and under LSTMWrapper)."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.exceptions import APIUsageError
from pufferlib_b200.frameworks import cleanrl
from framestack_oracle import FrameStackVec

pytestmark = pytest.mark.gpu

P = _native.ptr
FRAME = 84 * 84
Y_ROW = 32 * 400
INV255 = np.float32(1.0) / np.float32(255.0)
U = 2.0 ** -24
WG_CTAS = 264
GAME = {'pong': {'max_score': 2, 'max_ticks': 100}, 'breakout_pixels': {'max_ticks': 300}}
REFERENCE = {'frameskip': 4, 'noop_max': 30, 'episodic_life': True, 'clip_rewards': True}


def lib():
    return _native.lib()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def cpu(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def opts_of(kind, config):
    if config == 'plain':
        return {}
    o = dict(REFERENCE)
    if kind == 'pong':
        o.pop('episodic_life')
    return o


def iparam_of(kind, game):
    if kind == 'pong':
        return [game.get('max_score', 0), game.get('max_ticks', 0)]
    return [game.get('max_ticks', 0)]


def tape(kind, h, n, seed):
    if kind == 'pong':
        return np.random.default_rng(seed).integers(0, 6, size=(h, n)).astype(np.int64)
    return np.random.default_rng(seed).choice(4, size=(h, n), p=[0.2, 0.3, 0.25, 0.25]).astype(np.int64)


# ---- 1. the env against the one-frame oracle --------------------------------------------------------------------------
def check_step(t, got, want, infos=True):
    o, r, term, trunc, inf, _, mask = got
    oo, orr, ot, otr, oinf, _, om = want
    o = cpu(o)
    assert o.shape == oo.shape, (o.shape, oo.shape)
    if not np.array_equal(o, oo):
        bad = np.nonzero((o != oo).reshape(len(oo), -1).any(1))[0]
        raise AssertionError(f'step {t}: frames differ in envs {bad[:8]} ({len(bad)} envs)')
    assert np.array_equal(cpu(r).view(np.uint32), orr.view(np.uint32)), f'step {t}: reward bits differ'
    assert np.array_equal(cpu(term), ot), f'step {t}: terminals differ'
    assert np.array_equal(cpu(trunc), otr) and np.array_equal(cpu(mask), om), t
    if infos:
        assert len(inf) == len(oinf), (t, len(inf), len(oinf))
        for a, b in zip(inf, oinf):
            assert a == b, (t, a, b)


def compare_run(kind, n, h, seed, opts, game=None, offset=0, bound=False, host_buffers=False, infos=True, **make_kw):
    """Device at framestack=1 vs the one-frame oracle, every row of h steps and the reset row -> (game ends, nonzero
    rewards)."""
    game = GAME[kind] if game is None else game
    vec = pvec.make(ocean.env_creator(kind), env_kwargs={**game, **opts, 'framestack': 1}, num_envs=n,
                    backend=pvec.B200.options(exact_infos=infos, env_index_offset=offset, host_buffers=host_buffers),
                    **make_kw)
    assert vec.single_observation_space.shape == (1, 84, 84) and vec.obs_bytes == FRAME
    ora = FrameStackVec(kind, n, framestack=1, env_index_offset=offset, iparam=iparam_of(kind, game), **opts)
    acts = tape(kind, h, n, seed)
    vec.async_reset(seed)
    ora.async_reset(seed)
    exp = None
    if bound:
        exp = clean_pufferl.Experience(n * 8, 4, n * 8, (1, 84, 84), np.uint8, ())
        vec.bind_rollout(exp)
    ends = rewards = 0
    for t in range(h + 1):
        got = vec.recv()
        want = ora.recv()
        check_step(t, got, want, infos)
        ends += int(ora.ended.sum())
        rewards += int((want[1] != 0).sum())
        if t < h:
            a = torch.as_tensor(acts[t], device='cuda')
            if bound:
                z = torch.zeros(n, device='cuda')
                exp.store(got[0], z, a, z, got[1], got[2], got[5], got[6])
                if exp.full:
                    exp.sort_training_data()
            vec.send(a)
            ora.send(acts[t])
    vec.close()
    ora.close()
    return ends, rewards


@pytest.mark.parametrize('n', [1, 5, 33, 263])
@pytest.mark.parametrize('config', ['plain', 'reference'])
@pytest.mark.parametrize('kind', list(GAME))
def test_vs_oracle(kind, config, n):
    h = 400 if n <= 33 else 60
    opts = opts_of(kind, config)
    ends, rewards = compare_run(kind, n, h, 3 + n, opts)
    ticks = h * opts.get('frameskip', 1)        # breakout: bricks from about tick 60
    if n >= 5 and ticks >= 100:
        assert rewards > 0
    if n >= 5 and ticks > GAME[kind]['max_ticks'] + 30:
        assert ends > 0


@pytest.mark.parametrize('config', ['plain', 'reference'])
def test_every_ring_stage_wraps(config):
    """More than 4 x 2 x SMs envs, 30 sends: every CTA's 4-stage ring wraps several times per send, and each stage is
    rendered into again right behind its previous bulk store (the S = 1 ring's read wait)."""
    n = 4 * 2 * sms() * 3 + 37
    for kind in GAME:
        game = {'max_ticks': 40} if kind == 'breakout_pixels' else {'max_score': 2, 'max_ticks': 40}
        compare_run(kind, n, 30, 5, opts_of(kind, config), game=game, infos=False)


@pytest.mark.parametrize('config', ['plain', 'reference'])
@pytest.mark.parametrize('kind', list(GAME))
def test_bound_rollout_rows(kind, config):
    compare_run(kind, 33, 70, 5, opts_of(kind, config), bound=True)


@pytest.mark.parametrize('kind', list(GAME))
def test_host_buffers(kind):
    ends, _ = compare_run(kind, 33, 120, 6, opts_of(kind, 'reference'), host_buffers=True)
    assert ends > 0


def test_num_workers():
    compare_run('breakout_pixels', 32, 80, 8, REFERENCE, num_workers=2)
    compare_run('pong', 32, 80, 8, {}, num_workers=2)


def test_env_index_offset():
    compare_run('breakout_pixels', 16, 80, 9, REFERENCE, offset=1000)
    compare_run('pong', 16, 80, 9, {}, offset=12345)


@pytest.mark.parametrize('groups', [2, 4])
def test_pool_mode(groups):
    n, h, kind = 64, 60, 'breakout_pixels'
    b = n // groups
    vec = pvec.make(ocean.env_creator(kind), env_kwargs={**GAME[kind], **REFERENCE, 'framestack': 1}, num_envs=n,
                    backend=pvec.B200, batch_size=b)
    assert isinstance(vec, pvec.B200Pool)
    ora = FrameStackVec(kind, n, framestack=1, iparam=iparam_of(kind, GAME[kind]), **REFERENCE)
    acts = tape(kind, h, n, 4)
    vec.async_reset(7)
    ora.async_reset(7)
    for t in range(h):
        oo, orr, ot, _, _, _, _ = ora.recv()
        for g in range(groups):
            o, r, term, _, _, ids, _ = vec.recv()
            lo, hi = g * b, (g + 1) * b
            assert np.array_equal(ids, np.arange(lo, hi))
            assert np.array_equal(cpu(o), oo[lo:hi]) and np.array_equal(cpu(r), orr[lo:hi]), (t, g)
            assert np.array_equal(cpu(term), ot[lo:hi]), (t, g)
            vec.send(torch.as_tensor(acts[t, lo:hi], device='cuda'))
        ora.send(acts[t])
    vec.close()


# ---- 2. the env against itself ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('config', ['plain', 'reference'])
@pytest.mark.parametrize('kind', list(GAME))
def test_one_frame_is_the_newest_of_four(kind, config):
    n, h = 300, 340
    opts = {**GAME[kind], **opts_of(kind, config)}
    vecs = [pvec.make(ocean.env_creator(kind), env_kwargs={**opts, 'framestack': s}, num_envs=n,
                      backend=pvec.B200.options(exact_infos=True)) for s in (1, 4)]
    acts = tape(kind, h, n, 21)
    for v in vecs:
        v.async_reset(21)
    ends = 0
    for t in range(h + 1):
        (o1, r1, d1, tr1, i1, _, m1), (o4, r4, d4, tr4, i4, _, m4) = vecs[0].recv(), vecs[1].recv()
        assert o1.shape == (n, 1, 84, 84) and o4.shape == (n, 4, 84, 84)
        assert torch.equal(o1, o4[:, 3:]), t
        assert torch.equal(r1.view(torch.int32), r4.view(torch.int32)) and torch.equal(d1, d4), t
        assert torch.equal(tr1, tr4) and torch.equal(m1, m4) and i1 == i4, t
        ends += len(i1)
        if t < h:
            a = torch.as_tensor(acts[t], device='cuda')
            for v in vecs:
                v.send(a)
    assert vecs[0].episode_stats() == vecs[1].episode_stats()
    assert ends > 0
    for v in vecs:
        v.close()


# ---- 3. capture and refusals ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', list(GAME))
def test_captured_rollout_equals_eager(kind):
    n, h = 64, 40
    opts = {**GAME[kind], **opts_of(kind, 'reference'), 'framestack': 1}
    acts = torch.as_tensor(tape(kind, h, n, 3), device='cuda')

    def run(capture):
        vec = pvec.make(ocean.env_creator(kind), env_kwargs=opts, num_envs=n, backend=pvec.B200)
        vec.async_reset(11)
        vec.recv()
        vec.send(acts[0])
        vec.recv()
        torch.cuda.synchronize()
        obs = torch.zeros((h, n, 1, 84, 84), dtype=torch.uint8, device='cuda')
        rew = torch.zeros((h, n), device='cuda')
        term = torch.zeros((h, n), dtype=torch.bool, device='cuda')

        def body():
            for t in range(1, h):
                vec.send(acts[t])
                o, r, d, _, _, _, _ = vec.recv()
                obs[t].copy_(o)
                rew[t].copy_(r)
                term[t].copy_(d)
        if capture:
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                with torch.cuda.graph(g, stream=s):
                    body()
            torch.cuda.current_stream().wait_stream(s)
            g.replay()
        else:
            body()
        torch.cuda.synchronize()
        out = cpu(obs), cpu(rew), cpu(term)
        vec.close()
        return out
    eager, graph = run(False), run(True)
    for x, y in zip(eager, graph):
        assert np.array_equal(x, y)
    assert eager[2].any()


def test_env_refusals_launch_nothing():
    L = lib()
    for kind in GAME:
        for v in (2, 3, 5, -1, 8):
            iparam = [0] * 8
            iparam[6] = v
            cfg = _native.EnvConfig(kind=_native.ENV_KINDS[kind], num_envs=4, device=0, iparam=(C.c_int32 * 8)(*iparam))
            h = C.c_void_p()
            l0 = L.pb_launch_count()
            assert L.pb_env_create(C.byref(cfg), C.byref(h)) == _native.PB_ERR_INVALID, (kind, v)
            assert L.pb_launch_count() == l0 and not h.value, (kind, v)
            assert 'framestack' in _native.last_error()
        for kw in ({'framestack': 2}, {'framestack': True}, {'framestack': 1.0}):
            l0 = L.pb_launch_count()
            with pytest.raises(APIUsageError):
                pvec.make(ocean.env_creator(kind), env_kwargs=kw, num_envs=4, backend=pvec.B200)
            assert L.pb_launch_count() == l0
    with pytest.raises(APIUsageError):
        pvec.make(ocean.env_creator('breakout'), env_kwargs={'framestack': 1}, num_envs=4, backend=pvec.B200)


# ---- 4. conv1 at C = 1 ------------------------------------------------------------------------------------------------
def frames(m, stride, seed, c=1, poison_rows=2):
    """m rows of (c, 84, 84) uint8 `stride` bytes apart, then `poison_rows` rows of 255 never to be read; rows 0 and 1
    (when m > 2) all 0 and all 255."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    buf = torch.randint(0, 256, ((m + poison_rows) * stride,), dtype=torch.uint8, device='cuda', generator=gen)
    rows = buf.view(m + poison_rows, stride)
    rows[m:] = 255
    if m > 2:
        rows[0] = 0
        rows[1] = 255
    return torch.as_strided(buf, (m, c, 84, 84), (stride, FRAME, 84, 1))


def canaried(n, fill, extra=16):
    buf = torch.full((n + extra,), fill, dtype=torch.float32, device='cuda')
    return buf, buf[:n]


def fwd_ex(x, w, b, stream=None):
    c, m = x.shape[-3], x.shape[0] * (x.shape[1] * x.shape[2] if x.dim() == 6 else 1)
    yb, y = canaried(m * Y_ROW, -7.0)
    sp = _native.stream_ptr() if stream is None else stream
    if x.dim() == 6:
        _native.check(lib().pb_conv1_u8_forward_rows_ex(c, P(x), *segments(x), P(w), P(b), P(y), sp))
    else:
        _native.check(lib().pb_conv1_u8_forward_ex(c, P(x), x.stride(0), m, P(w), P(b), P(y), sp))
    assert bool((yb[m * Y_ROW:] == -7.0).all()), 'rows after y were written'
    return y.view(m, 32, 20, 20)


def wgrad_ex(x, y, dy):
    c, m = x.shape[-3], y.shape[0]
    dwb, dw = canaried(32 * 64 * c, float('nan'))
    dbb, db = canaried(32, float('nan'))
    nws = lib().pb_conv1_u8_wgrad_workspace_bytes(m)
    wsb = torch.full((nws + 64,), 0xA5, dtype=torch.uint8, device='cuda')
    if x.dim() == 6:
        _native.check(lib().pb_conv1_u8_wgrad_rows_ex(c, P(x), *segments(x), P(y), P(dy), P(dw), P(db), P(wsb), nws,
                                                      _native.stream_ptr()))
    else:
        _native.check(lib().pb_conv1_u8_wgrad_ex(c, P(x), x.stride(0), m, P(y), P(dy), P(dw), P(db), P(wsb), nws,
                                                 _native.stream_ptr()))
    assert bool(dwb[32 * 64 * c:].isnan().all()) and bool(dbb[32:].isnan().all()), 'elements after dw / db written'
    assert bool((wsb[nws:] == 0xA5).all()), 'bytes after the workspace were written'
    return dw.view(32, 64 * c), db


def segments(view):
    return view.shape[0] * view.shape[1], view.shape[2], view.shape[1], view.stride(0), view.stride(1), view.stride(2)


def cols64(x):
    return F.unfold(x.double(), 8, stride=4)      # [B, 64 c, 400]


def reduce_ref(parts):
    """k_reduce_partials in fp32: lane l sums partial rows l, l + 32, ... in order, then the xor tree."""
    lanes = np.zeros((32,) + parts.shape[1:], np.float32)
    for b_ in range(parts.shape[0]):
        lanes[b_ % 32] = lanes[b_ % 32] + parts[b_]
    for off in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ off]
    return lanes[0]


def grid_weights(seed, c=1):
    rng = np.random.default_rng(seed)
    w = rng.integers(-64, 65, (32, 64 * c)).astype(np.float32) / 256
    b = rng.integers(-64, 65, 32).astype(np.float32) / 256
    return torch.as_tensor(w, device='cuda'), torch.as_tensor(b, device='cuda')


def orthogonal_weights(seed, c=1):
    torch.manual_seed(seed)
    conv = models.layer_init(torch.nn.Conv2d(c, 32, 8, stride=4)).cuda()
    with torch.no_grad():
        conv.bias.uniform_(-0.5, 0.5)
    return conv.weight.detach().reshape(32, 64 * c).contiguous(), conv.bias.detach().clone()


@pytest.mark.parametrize('m', [1, 2, 3, 37, 263])
def test_exact_forward_and_wgrad_bitwise(m):
    """W, b, dy on the 2^-8 grid: every TF32 operand and every partial sum is exact, so y is relu(fl32(S * fl32(1/255)
    + b)) bit for bit, and with m <= 264 each weight-gradient CTA owns one row: its partial is fl32(S_row * fl32(1/255))
    (the in-CTA sum of the four pixel quarters is exact too), summed in k_reduce_partials' order."""
    w, b = grid_weights(m)
    x = frames(m, FRAME, seed=m)
    y = fwd_ex(x, w, b)
    xc = cols64(x)
    s = torch.einsum('ck,bkp->bcp', w.double(), xc)
    want = torch.relu((s * float(INV255) + b.double()[None, :, None]).float()).view(m, 32, 20, 20)
    assert torch.equal(y, want), float((y - want).abs().max())
    rng = np.random.default_rng(100 + m)
    dy = torch.as_tensor(rng.integers(-64, 65, (m, 32, 20, 20)).astype(np.float32) / 256, device='cuda')
    dw, db = wgrad_ex(x, y, dy)
    dz = (dy * (y > 0)).double().view(m, 32, 400)
    parts = (torch.einsum('bcp,bkp->bck', dz, xc) * float(INV255)).float().cpu().numpy().reshape(m, -1)
    assert np.array_equal(dw.cpu().numpy(), reduce_ref(parts).reshape(32, 64))
    assert torch.equal(db, dz.sum((0, 2)).float())


def check_general(m, stride, seed):
    """The module docstring's bounds of tests/test_gpu_nature_conv1.py at K = 64: 8 mma k-steps for the forward, 50 per
    row per CTA for the weight gradient (split into four quarters and summed in shared memory: 3 more adds)."""
    w, b = orthogonal_weights(seed)
    x = frames(m, stride, seed)
    y = fwd_ex(x, w, b)
    dy = torch.randn(m, 32, 20, 20, device='cuda', generator=torch.Generator(device='cuda').manual_seed(seed + 1))
    dw, db = wgrad_ex(x, y, dy)
    w64, wt = w.double(), w.double().abs()
    fwd_frac, dw64, dwabs, db64, dbabs = 0.0, 0, 0, 0, 0
    for lo in range(0, m, 4096):
        hi = min(m, lo + 4096)
        xc = cols64(x[lo:hi]) / 255.0
        ref = torch.relu(torch.einsum('ck,bkp->bcp', w64, xc) + b.double()[None, :, None])
        bound = (2.0 ** -11 + 16 * U) * torch.einsum('ck,bkp->bcp', wt, xc) + 2 * U * ref.abs() \
            + 2 * U * b.double().abs()[None, :, None] + 1e-30
        fwd_frac = max(fwd_frac, float(((y[lo:hi].view(hi - lo, 32, 400).double() - ref).abs() / bound).max()))
        dz = (dy[lo:hi] * (y[lo:hi] > 0)).double().view(hi - lo, 32, 400)
        dw64 = dw64 + torch.einsum('bcp,bkp->ck', dz, xc)
        dwabs = dwabs + torch.einsum('bcp,bkp->ck', dz.abs(), xc)
        db64 = db64 + dz.sum((0, 2))
        dbabs = dbabs + dz.abs().sum((0, 2))
    ctas = min(m, WG_CTAS)
    per_cta = -(-m // ctas)
    reduce_terms = -(-ctas // 32) + 16
    bw = (2.0 ** -11 + (50 * per_cta + 3 + reduce_terms) * U) * dwabs + 1e-30
    bb = (16 * per_cta + reduce_terms) * U * dbabs + 1e-30
    dw_frac = float(((dw.double() - dw64).abs() / bw).max())
    db_frac = float(((db.double() - db64).abs() / bb).max())
    print(f'C=1 m={m} stride={stride}: observed / bound  y {fwd_frac:.3f}  dW {dw_frac:.3f}  db {db_frac:.3f}', flush=True)
    assert fwd_frac <= 1.0 and dw_frac <= 1.0 and db_frac <= 1.0


def test_general_sizes_vs_fp64():
    g = 2 * sms()
    for m in (1, 2, 263, g + 1, 2 * g + 1, 4096):
        check_general(m, FRAME, seed=m % 97)
    check_general(263, FRAME + 16 * 7, seed=4)


def test_131072_rows_vs_fp64():
    check_general(131072, FRAME, seed=5)


def rollout_frames(envs, groups, steps, nm=2, mb=1, seed=0, outside=255):
    """An arrival-order one-frame rollout buffer [H*N, 1, 84, 84], the segment view [E, G, T, 1, 84, 84] of minibatch mb
    (Experience.segment_obs's strides) and its gathered copy; frames outside minibatch mb are `outside`."""
    horizon = steps * groups * nm
    gen = torch.Generator(device='cuda').manual_seed(seed)
    obs = torch.randint(0, 256, (horizon * envs, 1, 84, 84), dtype=torch.uint8, device='cuda', generator=gen)
    window = torch.arange(horizon, device='cuda') // steps
    obs.view(horizon, envs, FRAME)[window % nm != mb] = outside
    view = obs.view(groups, nm, steps, envs, 1, 84, 84)[:, mb].permute(2, 0, 1, 3, 4, 5)
    return obs, view, view.contiguous()


@pytest.mark.parametrize('steps', [1, 16])
@pytest.mark.parametrize('groups', [1, 4])
@pytest.mark.parametrize('envs', [1, 37])
def test_rows_bitwise_vs_dense_on_gathered_copy(envs, groups, steps):
    w, b = orthogonal_weights(envs * 7 + groups)
    _, view, gathered = rollout_frames(envs, groups, steps, seed=envs + 10 * groups + 100 * steps)
    m = envs * groups * steps
    x = gathered.view(m, 1, 84, 84)
    y_d, y_r = fwd_ex(x, w, b), fwd_ex(view, w, b)
    assert torch.equal(y_d, y_r)
    dy = torch.randn(m, 32, 20, 20, device='cuda', generator=torch.Generator(device='cuda').manual_seed(m))
    dw_d, db_d = wgrad_ex(x, y_d, dy)
    dw_r, db_r = wgrad_ex(view, y_r, dy)
    assert torch.equal(dw_d, dw_r) and torch.equal(db_d, db_r)
    _, view0, _ = rollout_frames(envs, groups, steps, seed=envs + 10 * groups + 100 * steps, outside=0)
    assert torch.equal(fwd_ex(view0, w, b), y_d)
    dw0, db0 = wgrad_ex(view0, y_r, dy)
    assert torch.equal(dw0, dw_d) and torch.equal(db0, db_d)


def test_deterministic_eager_and_graph():
    m = 4096
    w, b = orthogonal_weights(1)
    _, view, _ = rollout_frames(64, 2, 16, seed=1)
    x = frames(m, FRAME, 1)
    for inp in (x, view):
        y1, y2 = fwd_ex(inp, w, b), fwd_ex(inp, w, b)
        assert torch.equal(y1, y2)
        dy = torch.randn(m, 32, 20, 20, device='cuda')
        d1, d2 = wgrad_ex(inp, y1, dy), wgrad_ex(inp, y1, dy)
        assert torch.equal(d1[0], d2[0]) and torch.equal(d1[1], d2[1])
        yg, dwg, dbg = torch.empty_like(y1), torch.empty(32, 64, device='cuda'), torch.empty(32, device='cuda')
        ws = torch.empty(lib().pb_conv1_u8_wgrad_workspace_bytes(m), dtype=torch.uint8, device='cuda')
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                sp = _native.stream_ptr(s)
                if inp.dim() == 6:
                    _native.check(lib().pb_conv1_u8_forward_rows_ex(1, P(inp), *segments(inp), P(w), P(b), P(yg), sp))
                    _native.check(lib().pb_conv1_u8_wgrad_rows_ex(1, P(inp), *segments(inp), P(yg), P(dy), P(dwg),
                                                                  P(dbg), P(ws), ws.numel(), sp))
                else:
                    _native.check(lib().pb_conv1_u8_forward_ex(1, P(inp), FRAME, m, P(w), P(b), P(yg), sp))
                    _native.check(lib().pb_conv1_u8_wgrad_ex(1, P(inp), FRAME, m, P(yg), P(dy), P(dwg), P(dbg), P(ws),
                                                             ws.numel(), sp))
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(2):
            yg.zero_(), dwg.zero_(), dbg.zero_()
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(yg, y1) and torch.equal(dwg, d1[0]) and torch.equal(dbg, d1[1])


def test_ex_at_four_frames_is_the_existing_entry_points():
    m = 263
    w, b = orthogonal_weights(2, c=4)
    x = frames(m, 4 * FRAME, 2, c=4)
    y_old = torch.empty(m, 32, 20, 20, device='cuda')
    _native.check(lib().pb_conv1_u8_forward(P(x), x.stride(0), m, P(w), P(b), P(y_old), _native.stream_ptr()))
    y_new = fwd_ex(x, w, b)
    assert torch.equal(y_old, y_new)
    dy = torch.randn(m, 32, 20, 20, device='cuda')
    dw_old, db_old = torch.empty(32, 256, device='cuda'), torch.empty(32, device='cuda')
    nws = lib().pb_conv1_u8_wgrad_workspace_bytes(m)
    ws = torch.empty(nws, dtype=torch.uint8, device='cuda')
    _native.check(lib().pb_conv1_u8_wgrad(P(x), x.stride(0), m, P(y_old), P(dy), P(dw_old), P(db_old), P(ws), nws,
                                          _native.stream_ptr()))
    dw_new, db_new = wgrad_ex(x, y_new, dy)
    assert torch.equal(dw_old, dw_new) and torch.equal(db_old, db_new)
    obs = torch.randint(0, 256, (2 * 16 * 2 * 8, 4, 84, 84), dtype=torch.uint8, device='cuda')
    view = obs.view(2, 2, 16, 8, 4, 84, 84)[:, 1].permute(2, 0, 1, 3, 4, 5)
    ym = 8 * 2 * 16
    y_rows = torch.empty(ym, 32, 20, 20, device='cuda')
    _native.check(lib().pb_conv1_u8_forward_rows(P(view), *segments(view), P(w), P(b), P(y_rows), _native.stream_ptr()))
    assert torch.equal(y_rows, fwd_ex(view, w, b))


def test_ex_refusals_launch_nothing():
    L = lib()
    m = 8
    x1 = frames(m, FRAME, 0)
    w, b = orthogonal_weights(0)
    y = torch.empty(m, 32, 20, 20, device='cuda')
    dw, db = torch.empty(32, 256, device='cuda'), torch.empty(32, device='cuda')
    nws = L.pb_conv1_u8_wgrad_workspace_bytes(m)
    ws = torch.empty(nws, dtype=torch.uint8, device='cuda')
    sp = _native.stream_ptr()
    fwd = [(0, FRAME), (2, FRAME), (3, 3 * FRAME), (5, 5 * FRAME), (-1, FRAME), (1, FRAME - 16), (1, FRAME + 8),
           (4, FRAME), (4, 4 * FRAME - 16)]
    for frames_, stride in fwd:
        l0 = L.pb_launch_count()
        assert L.pb_conv1_u8_forward_ex(frames_, P(x1), stride, m, P(w), P(b), P(y), sp) == _native.PB_ERR_INVALID
        assert L.pb_conv1_u8_wgrad_ex(frames_, P(x1), stride, m, P(y), P(y), P(dw), P(db), P(ws), nws, sp) == \
            _native.PB_ERR_INVALID
        assert L.pb_launch_count() == l0, (frames_, stride)
    segs = [(2, FRAME, FRAME, FRAME), (1, FRAME - 16, FRAME, FRAME), (1, FRAME, FRAME + 8, FRAME),
            (1, FRAME, FRAME, FRAME - 16), (4, FRAME, FRAME, FRAME)]
    for frames_, se, sg, st in segs:
        l0 = L.pb_launch_count()
        assert L.pb_conv1_u8_forward_rows_ex(frames_, P(x1), 2, 4, 1, se, sg, st, P(w), P(b), P(y), sp) == \
            _native.PB_ERR_INVALID
        assert L.pb_conv1_u8_wgrad_rows_ex(frames_, P(x1), 2, 4, 1, se, sg, st, P(y), P(y), P(dw), P(db), P(ws), nws,
                                           sp) == _native.PB_ERR_INVALID
        assert L.pb_launch_count() == l0, (frames_, se, sg, st)


# ---- 5. the model and the trainer -------------------------------------------------------------------------------------
def fake_env(c):
    from test_gpu_policy_lstm import fake_env as fe
    return fe((c, 84, 84), 6, np.uint8)


def test_model_fast_vs_stock(monkeypatch):
    """Convolutional(framestack=1): the fast path against an fp64 restatement within the propagated bound of
    tests/test_gpu_nature_conv1.py (its conv1 bound taken at K = 256 is looser than K = 64 needs), and every gradient of
    a PPO minibatch within 1.5e-2 of each tensor's largest, against the stock path."""
    import pufferlib_b200
    from test_gpu_nature_conv1 import fp32_library_math, propagated_bound
    fp32_library_math(monkeypatch)
    torch.manual_seed(0)
    fast = models.Convolutional(fake_env(1), framestack=1).cuda()
    stock = models.Convolutional(fake_env(1), framestack=1).cuda()
    stock.load_state_dict(fast.state_dict())
    stock.fast_path = False
    x = frames(2048, FRAME, 3)
    calls = []
    orig = models._Conv1U8Function.apply
    monkeypatch.setattr(models._Conv1U8Function, 'apply', lambda *a: calls.append(1) or orig(*a))
    with torch.no_grad():
        lf, vf = fast(x[:512])
        (l64, bl), (v64, bv) = propagated_bound(stock, x[:512])
    assert len(calls) == 1
    assert float(((lf.double() - l64).abs() / (bl + 1e-30)).max()) <= 1.0
    assert float(((vf.double() - v64).abs() / (bv + 1e-30)).max()) <= 1.0
    m = 2048
    gen = torch.Generator(device='cuda').manual_seed(9)
    act = torch.randint(0, 6, (m,), device='cuda', generator=gen)
    old_lp = -torch.rand(m, device='cuda', generator=gen) - 1.0
    adv = torch.randn(m, device='cuda', generator=gen)
    ret, old_v = torch.randn(m, device='cuda', generator=gen), torch.randn(m, device='cuda', generator=gen)
    cfg = pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    grads = []
    for mdl in (fast, stock):
        logits, value = mdl(x)
        loss, _ = clean_pufferl.fused_ppo_loss(logits, value, act, old_lp, adv, ret, old_v, cfg)
        loss.backward()
        grads.append([p.grad.detach().clone() for p in mdl.parameters()])
    assert fast.network[0].weight.grad.shape == (32, 1, 8, 8)
    for (name, _), gf, gs in zip(fast.named_parameters(), *grads):
        frac = float((gf - gs).abs().max() / gs.abs().max())
        assert frac <= 1.5e-2, (name, frac)


@pytest.mark.parametrize('c', [2, 3])
def test_two_and_three_frames_run_the_stock_line(c, monkeypatch):
    torch.manual_seed(1)
    fast = models.Convolutional(fake_env(c), framestack=c).cuda()
    stock = models.Convolutional(fake_env(c), framestack=c).cuda()
    stock.load_state_dict(fast.state_dict())
    stock.fast_path = False
    x = frames(64, c * FRAME, 4, c=c)
    calls = []
    orig = models._Conv1U8Function.apply
    monkeypatch.setattr(models._Conv1U8Function, 'apply', lambda *a: calls.append(1) or orig(*a))
    with torch.no_grad():
        a, b_ = fast(x), stock(x)
    assert not calls
    assert torch.equal(a[0], b_[0]) and torch.equal(a[1], b_[1])


def trainer(kind, n, h, bptt, nm, recurrent, **kw):
    from test_gpu_config_updates import ppo_config
    vec = pvec.make(ocean.env_creator(kind), env_kwargs={'framestack': 1}, num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    if recurrent:
        net = models.LSTMWrapper(vec.driver_env, models.Convolutional(vec.driver_env, framestack=1), input_size=512,
                                 hidden_size=512)
        pol = cleanrl.RecurrentPolicy(net, seed=3).cuda()
        cfg = dict(fused_loss=True, learning_rate=2.5e-4, cuda_graph=True)
    else:
        pol = cleanrl.Policy(models.Convolutional(vec.driver_env, framestack=1), fused_sample=True, seed=3).cuda()
        cfg = dict(learning_rate=2.5e-4, cuda_graph=True)
    cfg.update(kw)
    return clean_pufferl.create(ppo_config(kind, n, h, bptt, nm, **cfg), vec, pol)


def plans_of(monkeypatch):
    plans = []
    update_plan = clean_pufferl.update_plan
    monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(update_plan(d)) or plans[-1])
    return plans


def test_convolutional_trains_on_one_frame(monkeypatch):
    plans = plans_of(monkeypatch)
    calls = []
    orig = models._Conv1U8Function.apply
    monkeypatch.setattr(models._Conv1U8Function, 'apply', lambda *a: calls.append(a[0].shape[-3]) or orig(*a))
    data = trainer('pong', 256, 32, 8, 2, False)
    for _ in range(3):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        assert np.isfinite([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy]).all()
    assert plans[-1].engine == 'model', plans[-1]
    assert data.graph_state == 2 and data.train_graph_state == 2, (data.graph_state, data.train_graph_state)
    assert calls and set(calls) == {1}
    clean_pufferl.close(data)


def loss_vector(data):
    return np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy, data.losses.approx_kl,
                     data.losses.clipfrac, data.losses.explained_variance])


@pytest.mark.parametrize('kind', list(GAME))
def test_conv_lstm_trains_on_one_frame(kind, monkeypatch):
    """LSTMWrapper(Convolutional(framestack=1)) at 256 x 32, bptt 8, 2 minibatches: plan ('cudnn_conv', 'segments',
    'whole') with both graphs captured; the captured update bitwise the eager one, and the segments form bitwise the
    gathered one, over two evaluate() + train() iterations from the same seeds."""
    plans = plans_of(monkeypatch)
    variants = {'captured': {}, 'eager': dict(cuda_graph_train=False),
                'gathered': dict(cuda_graph_train=False, zero_copy_minibatches=False)}
    expect = {'captured': ('cudnn_conv', 'segments', 'whole'), 'eager': ('cudnn_conv', 'segments', None),
              'gathered': ('cudnn_conv', 'gathered', None)}
    res = {}
    for name, kw in variants.items():
        data = trainer(kind, 256, 32, 8, 2, True, **kw)
        out = []
        for _ in range(2):
            clean_pufferl.evaluate(data)
            clean_pufferl.train(data)
            p = plans[-1]
            assert (p.engine, p.form, p.capture) == expect[name], (name, p)
            assert np.isfinite(loss_vector(data)[:5]).all(), name
            out.append(({k: q.detach().clone() for k, q in data.policy.named_parameters()}, loss_vector(data)))
        if name == 'captured':
            assert data.graph_state == 2 and data.train_graph_state == 2, (data.graph_state, data.train_graph_state)
        res[name] = out
        clean_pufferl.close(data)
    for a_, b_ in (('captured', 'eager'), ('eager', 'gathered')):
        for it in range(2):
            assert np.array_equal(res[a_][it][1], res[b_][it][1], equal_nan=True), (a_, b_, it)
            for k, v in res[a_][it][0].items():
                assert torch.equal(v, res[b_][it][0][k]), (a_, b_, it, k)


def test_pong_one_frame_full_size_within_budget(monkeypatch):
    """pong at 4 096 envs x 128 steps, bptt 16, 4 minibatches: the rollout holds one frame per row (7 056 bytes), and the
    peak stays under the C4 budget of tests/test_gpu_conv_lstm.py with that row size."""
    plans = plans_of(monkeypatch)
    n, h, nm = 4096, 128, 4
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    data = trainer('pong', n, h, 16, nm, True)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        assert np.isfinite(loss_vector(data)[:5]).all()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    mb = n * h // nm
    budget = n * h * FRAME + mb * 4 * (2 * Y_ROW + 3 * (5184 + 3136 + 512) + 12 * 512) + 4 * 2 ** 30
    print(f'pong one-frame C4 LSTM(Conv): peak {peak / 2 ** 30:.2f} GiB, budget {budget / 2 ** 30:.2f} GiB, '
          f'graph states {data.graph_state} / {data.train_graph_state}', flush=True)
    assert (plans[-1].engine, plans[-1].form) == ('cudnn_conv', 'segments')
    assert data.experience.obs.shape[1:] == (1, 84, 84) and data.experience._b_obs is None
    assert peak <= budget
    clean_pufferl.close(data)
