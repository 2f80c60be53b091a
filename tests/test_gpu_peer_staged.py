"""The multi-GPU gradient exchange (csrc/peer.cu, peer.cuh) and the optimizer kernels that contain it (csrc/optim.cu), run as
ONE rank of a world of up to 8 on one device against peers staged by the test (tests/util_peer.py).

The exchange must equal the fp32 sum of the ranks' gradients in rank order bit for bit, advance the epoch counter by one, and
leave exactly the protocol's bytes in all W peer buffers; the fused exchange + clip + Adam kernels must equal the
single-rank kernels run on that sum bit for bit, and clip_grad_norm_ + torch.optim.Adam to fp32 noise.  This covers the
arithmetic and the addresses of the protocol.  It says nothing about the visibility of stores between devices or the IPC
mapping: those need several GPUs (tests/multi_gpu/check_peer_update.py).

No test here lets a kernel wait: every launch that polls flags is made by StagedPeers.exchange / replay, after the flags
are written.
"""
import ctypes as C

import pytest
import torch

from pufferlib_b200 import _native
from pufferlib_b200.exceptions import APIUsageError

import util_peer as up

pytestmark = pytest.mark.gpu

WORLDS = [(2, 0), (2, 1), (3, 1), (4, 3), (8, 0), (8, 5), (8, 7)]
# 514 = models.Default's 1-feature, 1-action parameters back to back, 17157 breakout's, 17415 six actions'; below 900 the
# trailing slices of the 16-slice form are empty; 1, 3, 5, 514, 771, 899 end in a scalar tail (n % 4 != 0)
SIZES = [1, 3, 4, 5, 514, 771, 899, 900, 17157, 17415, 20000]
BETAS_EPS = (C.c_float(0.9), C.c_float(0.999), C.c_float(1e-5))
LR, MAX_NORM = 2.5e-4, 0.5


def round4(n):
    return (n + 3) // 4 * 4


def buffer_cases():
    """(n, capacity, flat 4 bytes past a 16-byte boundary): the slot filled to the end and with 8 spare floats (both keep
    the 128-bit path), and for two sizes a capacity that is no multiple of 4 and a misaligned flat buffer (both force the
    scalar path)."""
    for n in SIZES:
        yield pytest.param(n, round4(n), False, id=f'n{n}-tight')
        yield pytest.param(n, round4(n) + 8, False, id=f'n{n}-slack')
    for n in (5, 17157):
        yield pytest.param(n, round4(n) + 1, False, id=f'n{n}-oddcap')
        yield pytest.param(n, round4(n), True, id=f'n{n}-offset')


def flat_buffer(n, offset, dev):
    """-> (the n-float view the kernel sums in place, the floats before and after it in its storage: all 7.0)."""
    store = torch.full((n + 8,), 7.0, device=dev)
    assert store.data_ptr() % 16 == 0
    lo = 4 + int(offset)
    flat = store[lo:lo + n]
    assert flat.data_ptr() % 16 == (4 if offset else 0)
    return flat, (store[:lo], store[lo + n:])


def check_sum(flat, g, around):
    want = up.rank_order_sum(g)
    assert torch.equal(up.bits(flat), up.bits(want)), \
        f'{int((up.bits(flat) != up.bits(want)).sum())} of {flat.numel()} elements differ from the fp32 sum in rank order'
    # the reference itself against fp64: W roundings of at most 2^-24 of a partial sum each
    g64 = g.double()
    assert bool(((want.double() - g64.sum(0)).abs() <= 1e-6 * g64.abs().sum(0)).all())
    assert all(bool((t == 7.0).all()) for t in around), 'a store outside flat[0, n)'
    return want


@pytest.mark.parametrize('n,capacity,offset', list(buffer_cases()))
@pytest.mark.parametrize('world,rank', WORLDS)
def test_peer_allreduce_is_the_rank_order_sum(world, rank, n, capacity, offset):
    """pb_peer_allreduce (one CTA), three calls in a row: epochs 1, 2, 3, so slot 1, slot 0 and slot 1 again."""
    dev = torch.device('cuda')
    lib, s = _native.lib(), _native.stream_ptr()
    peers = up.StagedPeers(world, rank, capacity, dev, sliced=False)
    flat, around = flat_buffer(n, offset, dev)
    for call in range(3):
        g = up.gradients(n, world, 1000 * n + 10 * world + call, dev)
        flat.copy_(g[rank])
        e = peers.exchange(flat, g, lambda comm: _native.check(lib.pb_peer_allreduce(C.byref(comm), _native.ptr(flat), n, s)))
        assert e == call + 1
        check_sum(flat, g, around)
        peers.check_epoch()
        peers.check_buffers()


@pytest.mark.parametrize('n,capacity,offset', list(buffer_cases()))
@pytest.mark.parametrize('world,rank', WORLDS)
def test_peer_allreduce_parts_sums_every_element_once(world, rank, n, capacity, offset):
    """pb_peer_allreduce_parts (16 CTAs, one slice each) followed by pb_clip_adam_parts(..., peer_epoch), three times.  The
    16 partial sums of squares are the check that no element is summed by two slices or by none: each must be the fp64 sum of
    squares of its slice of the summed gradient, an empty slice exactly 0."""
    dev = torch.device('cuda')
    lib, s = _native.lib(), _native.stream_ptr()
    assert lib.pb_peer_slices() == up.SLICES
    peers = up.StagedPeers(world, rank, capacity, dev, sliced=True)
    flat, around = flat_buffer(n, offset, dev)
    parts = torch.full((up.SLICES,), float('nan'), dtype=torch.float64, device=dev)
    p, m, v, step = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros((), device=dev)
    arr = (_native.AdamTensor * 1)(_native.AdamTensor(p.data_ptr(), m.data_ptr(), v.data_ptr(), step.data_ptr(), flat.data_ptr(), n))
    bounds = up.slice_bounds(n)
    assert bounds[0][0] == 0 and bounds[-1][1] == n and all(a[1] == b[0] and (b[0] % 4 == 0 or b[0] == n) for a, b in zip(bounds, bounds[1:]))
    for call in range(3):
        g = up.gradients(n, world, 1000 * n + 10 * world + call, dev)
        flat.copy_(g[rank])
        parts.fill_(float('nan'))
        peers.exchange(flat, g, lambda comm: _native.check(lib.pb_peer_allreduce_parts(
            C.byref(comm), _native.ptr(flat), n, _native.ptr(parts), s)), advances=False)
        peers.check_epoch()                  # the sliced exchange leaves the counter alone ...
        _native.check(lib.pb_clip_adam_parts(arr, 1, C.c_float(MAX_NORM), C.c_float(1.0 / world), C.c_float(LR), None, *BETAS_EPS,
                                             None, _native.ptr(parts), up.SLICES, _native.ptr(peers.epoch_dev), None, s))
        peers.advanced()
        peers.check_epoch()                  # ... and the optimizer kernel that follows advances it by one
        want = check_sum(flat, g, around)
        peers.check_buffers()
        assert float(step) == call + 1
        sq = want.double() ** 2
        got = parts.cpu()
        for b, (lo, hi) in enumerate(bounds):
            ref = float(sq[lo:hi].sum())
            if lo == hi:
                assert float(got[b]) == 0.0, f'slice {b} of n = {n} is empty but its sum of squares is {float(got[b])!r}'
            else:
                assert abs(float(got[b]) - ref) <= 1e-12 * ref, (b, lo, hi, float(got[b]), ref)
        total = float(sq.sum())
        assert abs(float(got.sum()) - total) <= 1e-12 * total, (float(got.sum()), total)


# ---- the optimizer step as train() runs it

def default_layout(features, n_act, layout):
    """Where the gradients of models.Default's six parameters (encoder weight and bias, decoder weight and bias, value weight
    and bias) lie in the flat buffer -> (n, [(offset, numel)] * 6).  'update': _DefaultMLPUpdate's buffer, dW_enc | 8 head
    rows x 128 | db_enc | 8 head biases, whose padding rows hold zeros.  'packed': the six gradients back to back, which the C
    ABI accepts as well and which gives buffer sizes that are no multiple of 4."""
    hid = 128
    if layout == 'packed':
        sizes = [hid * features, hid, n_act * hid, n_act, hid, 1]
        offs = [sum(sizes[:i]) for i in range(6)]
        return sum(sizes), list(zip(offs, sizes))
    w_cat, b_enc, b_cat = hid * features, hid * features + 8 * hid, hid * features + 9 * hid
    return b_cat + 8, [(0, hid * features), (b_enc, hid), (w_cat, n_act * hid), (b_cat, n_act), (w_cat + n_act * hid, hid),
                       (b_cat + n_act, 1)]


class Engine:
    """One copy of the parameters, Adam state, flat gradient buffer and head matrix."""

    def __init__(self, params, n, views, n_act, dev):
        self.p = [q.clone() for q in params]
        self.m, self.v = [torch.zeros_like(q) for q in params], [torch.zeros_like(q) for q in params]
        self.step = [torch.zeros((), device=dev) for _ in params]
        self.flat = torch.zeros(n, device=dev)
        self.grads = [self.flat[o:o + k] for o, k in views]
        self.arr = (_native.AdamTensor * 6)()
        for i in range(6):
            self.arr[i] = _native.AdamTensor(self.p[i].data_ptr(), self.m[i].data_ptr(), self.v[i].data_ptr(),
                                             self.step[i].data_ptr(), self.grads[i].data_ptr(), self.p[i].numel())
        self.norm = torch.zeros(1, device=dev)
        self.w_cat, self.b_cat = torch.zeros(8, 128, device=dev), torch.zeros(8, device=dev)
        self.n_act = n_act
        self.pack = _native.HeadPack(self.p[2].data_ptr(), self.p[3].data_ptr(), self.p[4].data_ptr(), self.p[5].data_ptr(),
                                     self.w_cat.data_ptr(), self.b_cat.data_ptr(), n_act, 128)
        self.parts = torch.zeros(up.SLICES, dtype=torch.float64, device=dev)

    def hyper(self, world, lr_t):
        return (C.c_float(MAX_NORM), C.c_float(1.0 / world), C.c_float(0.0 if lr_t is not None else LR), _native.ptr(lr_t),
                *BETAS_EPS, _native.ptr(self.norm))

    def packed_heads(self):
        w, b = torch.full_like(self.w_cat, 9.0), torch.full_like(self.b_cat, 9.0)
        _native.check(_native.lib().pb_pack_heads(_native.ptr(self.p[2]), _native.ptr(self.p[3]), _native.ptr(self.p[4]),
                                                  _native.ptr(self.p[5]), self.n_act, 128, _native.ptr(w), _native.ptr(b), None,
                                                  None, 0, _native.stream_ptr()))
        return w, b

    def state(self):
        return self.p + self.m + self.v + self.step + [self.norm]


def assert_same_bits(a, b, what):
    names = [f'{kind}[{i}]' for kind in ('param', 'exp_avg', 'exp_avg_sq', 'step') for i in range(6)] + ['total_norm']
    for name, x, y in zip(names, a.state(), b.state()):
        assert torch.equal(up.bits(x), up.bits(y)), f'{what}: {name} differs in {int((up.bits(x) != up.bits(y)).sum())} elements'


def default_parameters(features, n_act, dev):
    """Six separate allocations, as the nn.Linear weights and biases of a models.Default are."""
    shapes = [(128, features), (128,), (n_act, 128), (n_act,), (1, 128), (1,)]
    return [torch.randn(s, device=dev) * 0.1 for s in shapes]


def step_gradients(n, views, world, seed, dev):
    """Five steps of per-rank gradients [W, n]: zero outside the six views, scaled so that the mean gradient's norm is about
    0.1 (no clipping at max_norm 0.5), and 200 times that on step 2 (clipped)."""
    mask = torch.zeros(n, device=dev)
    for o, k in views:
        mask[o:o + k] = 1.0
    first = up.gradients(n, world, seed, dev) * mask
    scale = 0.1 / float((first.double().sum(0) / world).norm())
    return [up.gradients(n, world, seed + it, dev, scale * (200.0 if it == 2 else 1.0)) * mask for it in range(5)]


class TorchAdam:
    """clip_grad_norm_ + torch.optim.Adam(eps=1e-5, fused, capturable) on the summed gradient divided by the world size."""

    def __init__(self, params, views, world, lr_t):
        self.ref = [q.clone().requires_grad_(True) for q in params]
        self.opt = torch.optim.Adam(self.ref, lr=lr_t.clone() if lr_t is not None else LR, eps=1e-5, fused=True, capturable=True)
        self.views, self.world = views, world

    def step(self, summed):
        for q, (o, k) in zip(self.ref, self.views):
            q.grad = (summed[o:o + k] / self.world).view_as(q).clone()
        norm = float(torch.nn.utils.clip_grad_norm_(self.ref, MAX_NORM))
        self.opt.step()
        return norm

    def check(self, eng, norm, it):
        assert abs(float(eng.norm) - norm) <= 1e-5 * norm, (it, float(eng.norm), norm)
        for i, q in enumerate(self.ref):
            st = self.opt.state[q]
            assert float(eng.step[i]) == float(st['step']) == it + 1
            for mine, theirs in ((eng.m[i], st['exp_avg']), (eng.v[i], st['exp_avg_sq'])):
                assert torch.allclose(mine, theirs, rtol=1e-5, atol=1e-6 * float(theirs.abs().max())), (it, i)
            assert float((eng.p[i] - q.detach()).abs().max()) <= 1e-3 * LR * (it + 1), (it, i)


# world, rank (first and last), learning rate through lr_dev
STEP_WORLDS = [(2, 0, False), (2, 1, True), (4, 0, True), (4, 3, False), (8, 0, False), (8, 7, True)]
# features, actions, layout: breakout and six actions, the ocean envs' 1 x 1 and 7 x 2; n = 17157, 17415, 514, 1411 packed,
# 17544 and 1288 as _DefaultMLPUpdate lays the buffer out
STEP_SHAPES = [(128, 4, 'packed'), (128, 6, 'packed'), (1, 1, 'packed'), (7, 2, 'packed'), (128, 4, 'update'), (1, 1, 'update')]


@pytest.mark.parametrize('features,n_act,layout', STEP_SHAPES)
@pytest.mark.parametrize('world,rank,lr_on_device', STEP_WORLDS)
def test_clip_adam_peer_is_clip_adam_on_the_rank_order_sum(world, rank, lr_on_device, features, n_act, layout):
    """pb_clip_adam_peer (one CTA: exchange, norm pass, clip, Adam) against staged peers, five steps, vs pb_clip_adam on the
    rank-order sum formed by the test (the same kernel body on the same bits: everything bitwise equal) and vs torch."""
    dev = torch.device('cuda')
    torch.manual_seed(7)
    lib, s = _native.lib(), _native.stream_ptr()
    n, views = default_layout(features, n_act, layout)
    params = default_parameters(features, n_act, dev)
    lr_t = torch.tensor(LR, device=dev) if lr_on_device else None
    fused, plain = Engine(params, n, views, n_act, dev), Engine(params, n, views, n_act, dev)
    ref = TorchAdam(params, views, world, lr_t)
    peers = up.StagedPeers(world, rank, round4(n), dev, sliced=False)
    for it, g in enumerate(step_gradients(n, views, world, 100 * features + n_act, dev)):
        summed = up.rank_order_sum(g)
        fused.flat.copy_(g[rank])
        peers.exchange(fused.flat, g, lambda comm: _native.check(lib.pb_clip_adam_peer(
            fused.arr, 6, *fused.hyper(world, lr_t), C.byref(comm), _native.ptr(fused.flat), n, s)))
        plain.flat.copy_(summed)
        _native.check(lib.pb_clip_adam(plain.arr, 6, *plain.hyper(world, lr_t), s))
        norm = ref.step(summed)
        assert (norm > MAX_NORM) == (it == 2), (it, norm)
        peers.check_epoch()
        peers.check_buffers()
        assert torch.equal(up.bits(fused.flat), up.bits(summed))
        assert_same_bits(fused, plain, f'step {it}, pb_clip_adam_peer vs pb_clip_adam on the sum')
        ref.check(fused, norm, it)


@pytest.mark.parametrize('with_pack', [True, False])
@pytest.mark.parametrize('features,n_act,layout', STEP_SHAPES)
@pytest.mark.parametrize('world,rank,lr_on_device', STEP_WORLDS)
def test_clip_adam_peer_parts_is_the_two_kernel_pair(world, rank, lr_on_device, features, n_act, layout, with_pack):
    """pb_clip_adam_peer_parts, the kernel _DefaultMLPUpdate.optimizer_step launches on several GPUs (16 CTAs of 512 threads:
    sliced exchange, grid barrier, clip, Adam, epoch advance, head matrix rebuilt by the last CTA), five steps, vs the pair
    pb_peer_allreduce_parts + pb_clip_adam_parts with 16 parts (32 CTAs of 256 threads).  Both sum the same 16 partial sums
    in the same order and apply the same per-element update, so parameters, moments, step counters and the norm are bitwise
    equal; vs torch to fp32 noise.  With a head pack, w_cat / b_cat must equal pb_pack_heads of the updated parameters: the
    last CTA reads head parameters that other CTAs of the launch have just written."""
    dev = torch.device('cuda')
    torch.manual_seed(7)
    lib, s = _native.lib(), _native.stream_ptr()
    n, views = default_layout(features, n_act, layout)
    params = default_parameters(features, n_act, dev)
    lr_t = torch.tensor(LR, device=dev) if lr_on_device else None
    fused, pair = Engine(params, n, views, n_act, dev), Engine(params, n, views, n_act, dev)
    ref = TorchAdam(params, views, world, lr_t)
    peers_f = up.StagedPeers(world, rank, round4(n), dev, sliced=True)
    peers_p = up.StagedPeers(world, rank, round4(n), dev, sliced=True)
    for it, g in enumerate(step_gradients(n, views, world, 100 * features + n_act, dev)):
        summed = up.rank_order_sum(g)
        for eng in (fused, pair):
            eng.flat.copy_(g[rank])
            eng.w_cat.fill_(9.0)
            eng.b_cat.fill_(9.0)
        peers_f.exchange(fused.flat, g, lambda comm: _native.check(lib.pb_clip_adam_peer_parts(
            fused.arr, 6, *fused.hyper(world, lr_t), C.byref(comm), _native.ptr(fused.flat), n, _native.ptr(fused.parts),
            C.byref(fused.pack) if with_pack else None, s)))
        peers_p.exchange(pair.flat, g, lambda comm: _native.check(lib.pb_peer_allreduce_parts(
            C.byref(comm), _native.ptr(pair.flat), n, _native.ptr(pair.parts), s)), advances=False)
        _native.check(lib.pb_clip_adam_parts(pair.arr, 6, *pair.hyper(world, lr_t), _native.ptr(pair.parts), up.SLICES,
                                             _native.ptr(peers_p.epoch_dev), C.byref(pair.pack) if with_pack else None, s))
        peers_p.advanced()
        norm = ref.step(summed)
        assert (norm > MAX_NORM) == (it == 2), (it, norm)
        for peers in (peers_f, peers_p):
            peers.check_epoch()
            peers.check_buffers()
        assert torch.equal(up.bits(fused.flat), up.bits(summed))
        assert torch.equal(fused.parts, pair.parts)
        total = float((summed.double() ** 2).sum())
        assert abs(float(fused.parts.sum()) - total) <= 1e-12 * total
        assert_same_bits(fused, pair, f'step {it}, pb_clip_adam_peer_parts vs pb_peer_allreduce_parts + pb_clip_adam_parts')
        ref.check(fused, norm, it)
        for eng in (fused, pair):
            if with_pack:
                w_ref, b_ref = eng.packed_heads()
                assert torch.equal(eng.w_cat, w_ref) and torch.equal(eng.b_cat, b_ref), it
            else:
                assert bool((eng.w_cat == 9.0).all()) and bool((eng.b_cat == 9.0).all())


@pytest.mark.parametrize('world,rank,features,n_act,layout', [(2, 1, 128, 4, 'update'), (8, 0, 1, 1, 'packed'), (4, 3, 7, 2, 'packed')])
def test_clip_adam_peer_parts_replays_in_a_graph(world, rank, features, n_act, layout):
    """Three pb_clip_adam_peer_parts steps captured in one CUDA graph, as train() captures the whole update, replayed twice
    (epochs 1-3 and 4-6) vs the same six steps run eagerly from the same start.  Before a replay both slots of every peer are
    staged (one gradient set per epoch parity) and every peer flag is set to the last epoch the replay reaches."""
    dev = torch.device('cuda')
    torch.manual_seed(11)
    lib = _native.lib()
    n, views = default_layout(features, n_act, layout)
    params = default_parameters(features, n_act, dev)
    lr_t = torch.tensor(LR, device=dev)
    sets = step_gradients(n, views, world, 500 + features, dev)
    by_parity = sets[:2]
    own = [sets[3][0], sets[2][0], sets[4][0]]          # three own gradients; the second is 200 times larger: clipped
    eager, graphed = Engine(params, n, views, n_act, dev), Engine(params, n, views, n_act, dev)

    def step(eng, comm):
        _native.check(lib.pb_clip_adam_peer_parts(eng.arr, 6, *eng.hyper(world, lr_t), C.byref(comm), _native.ptr(eng.flat), n,
                                                  _native.ptr(eng.parts), C.byref(eng.pack), _native.stream_ptr()))

    def three_steps(comm):
        for it in range(3):
            graphed.flat.copy_(own[it])
            step(graphed, comm)

    peers_e = up.StagedPeers(world, rank, round4(n), dev, sliced=True)
    after = []
    for it in range(6):
        eager.flat.copy_(own[it % 3])
        peers_e.exchange(eager.flat, by_parity[(it + 1) & 1], lambda comm: step(eager, comm))
        if it % 3 == 2:
            after.append([t.clone() for t in eager.state() + [eager.w_cat, eager.b_cat]])
    peers_e.check_epoch()

    peers_g = up.StagedPeers(world, rank, round4(n), dev, sliced=True)
    graph = peers_g.capture(three_steps)
    for replay in range(2):
        peers_g.replay(graph, by_parity, n, 3)
        torch.cuda.synchronize()
        peers_g.check_epoch()
        assert peers_g.epoch == 3 * (replay + 1)
        for name, x, y in zip(range(99), graphed.state() + [graphed.w_cat, graphed.b_cat], after[replay]):
            assert torch.equal(up.bits(x), up.bits(y)), (replay, name)


# ---- argument checks

def raised_world(dev, capacity=64):
    """An 8-rank communicator in which every flag of every buffer is far ahead of the epoch: every call of the test below is
    refused on the host before any launch, and if a check stopped firing the kernel would run through instead of waiting."""
    peers = up.StagedPeers(8, 0, capacity, dev, sliced=True)
    for buf in peers.bufs:
        buf[:up.HEADER_WORDS] = 1 << 40
    return peers


def comm_with(peers, **changes):
    c = _native.PeerComm.from_buffer_copy(peers.struct)
    for key, value in changes.items():
        if key.startswith('base'):
            c.base[int(key[4:])] = value
        else:
            setattr(c, key, value)
    return c


def test_peer_argument_checks():
    dev = torch.device('cuda')
    lib, s = _native.lib(), _native.stream_ptr()
    for c in (1, 4, 17157, 20000):
        assert lib.pb_peer_buffer_bytes(c) == 1024 + 8 * c
    assert lib.pb_peer_slices() == 16
    peers = raised_world(dev)                  # buffers of 64 floats per slot; the communicators below claim 16
    n, views = 16, [(0, 4), (4, 4), (8, 2), (10, 2), (12, 2), (14, 2)]
    eng = Engine([torch.zeros(k, device=dev) for _, k in views], n, views, 2, dev)
    hyper = eng.hyper(8, None)
    launches = lib.pb_launch_count()
    bad = [('world = 9', dict(world=9), n), ('rank = world', dict(rank=8), n), ('negative rank', dict(rank=-1), n),
           ('n > capacity', {}, 17), ('null base', dict(base5=None), n), ('null epoch', dict(epoch=None), n)]
    for what, changes, count in bad:
        comm = comm_with(peers, capacity=16, **changes)
        calls = {
            'pb_peer_allreduce': lambda: lib.pb_peer_allreduce(C.byref(comm), _native.ptr(eng.flat), count, s),
            'pb_peer_allreduce_parts': lambda: lib.pb_peer_allreduce_parts(C.byref(comm), _native.ptr(eng.flat), count,
                                                                           _native.ptr(eng.parts), s),
            'pb_clip_adam_peer': lambda: lib.pb_clip_adam_peer(eng.arr, 6, *hyper, C.byref(comm), _native.ptr(eng.flat), count, s),
            'pb_clip_adam_peer_parts': lambda: lib.pb_clip_adam_peer_parts(eng.arr, 6, *hyper, C.byref(comm), _native.ptr(eng.flat),
                                                                           count, _native.ptr(eng.parts), None, s),
        }
        for name, call in calls.items():
            with pytest.raises(APIUsageError, match=f'^{name}: '):
                _native.check(call())
            assert lib.pb_launch_count() == launches, (what, name)
    # a gradient view that is not inside the flat buffer
    comm = comm_with(peers, capacity=16)
    elsewhere = torch.zeros(4, device=dev)
    eng.arr[1].grad = elsewhere.data_ptr()
    with pytest.raises(APIUsageError, match='outside the flat buffer'):
        _native.check(lib.pb_clip_adam_peer(eng.arr, 6, *hyper, C.byref(comm), _native.ptr(eng.flat), n, s))
    with pytest.raises(APIUsageError, match='outside the flat buffer'):
        _native.check(lib.pb_clip_adam_peer_parts(eng.arr, 6, *hyper, C.byref(comm), _native.ptr(eng.flat), n,
                                                  _native.ptr(eng.parts), None, s))
    eng.arr[1].grad = eng.grads[1].data_ptr()
    # the fused sliced kernel is for several ranks only
    with pytest.raises(APIUsageError):
        _native.check(lib.pb_clip_adam_peer_parts(eng.arr, 6, *hyper, C.byref(comm_with(peers, capacity=16, world=1)),
                                                  _native.ptr(eng.flat), n, _native.ptr(eng.parts), None, s))
    assert lib.pb_launch_count() == launches   # nothing ran
    peers.check_epoch()


@pytest.mark.parametrize('single', ['no communicator', 'world = 1'])
def test_clip_adam_peer_without_peers_is_clip_adam(single):
    """pb_clip_adam_peer with comm = NULL or a world of one rank is pb_clip_adam: same bits, no buffer touched, no epoch."""
    dev = torch.device('cuda')
    torch.manual_seed(5)
    lib, s = _native.lib(), _native.stream_ptr()
    n, views = default_layout(7, 2, 'packed')
    params = default_parameters(7, 2, dev)
    a, b = Engine(params, n, views, 2, dev), Engine(params, n, views, 2, dev)
    peers = up.StagedPeers(2, 0, round4(n), dev, sliced=False)
    comm = comm_with(peers, world=1)
    for it, g in enumerate(step_gradients(n, views, 1, 3, dev)):
        a.flat.copy_(g[0])
        b.flat.copy_(g[0])
        _native.check(lib.pb_clip_adam_peer(a.arr, 6, *a.hyper(1, None), C.byref(comm) if single == 'world = 1' else None,
                                            _native.ptr(a.flat), n, s))
        _native.check(lib.pb_clip_adam(b.arr, 6, *b.hyper(1, None), s))
        assert_same_bits(a, b, f'step {it}')
        assert torch.equal(up.bits(a.flat), up.bits(g[0]))
    peers.check_epoch()
    peers.check_buffers()
