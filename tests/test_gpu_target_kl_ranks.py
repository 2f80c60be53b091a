"""target_kl on several ranks, on ONE device against staged peers (tests/util_peer.py): the KL row sum carried by the
gradient exchange (pb_clip_adam_peer_ex / pb_clip_adam_peer_parts_ex), the stop decided on it by pb_kl_stop with
rows = world * rows per minibatch, and train() playing rank k of 2 with the communicator replaced by the staged one.

1. Kernels.  With a payload, both _ex kernels leave the summed gradient, parameters, moments, steps, head matrix and norm
   bitwise equal to the existing entry points on the same staged gradients (the payloads are about 1e30, so one that leaked
   into the norm would show), *kl_out bitwise equal to the fp64 sum of the payloads in rank order, and every byte of all W
   buffers as the protocol says.  The existing entry points leave the payload floats' NaN canaries alone.  A captured graph
   of several exchanges replays like the eager ones; the argument checks refuse before any launch.
2. The decision: on the KL sum over the ranks, the same at every own-rank position.
3. train(): epochs run as the mean over the ranks decides, captured equal to eager, the device epoch counter advanced by
   exactly the exchanges that ran.

No test here lets a kernel wait: every launch that polls flags is staged first (StagedPeers.exchange / replay, or
KLPeers.stage_ahead before a train() call, which stages every exchange the call can make).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.exceptions import APIUsageError
from pufferlib_b200.frameworks import cleanrl

import util_peer as up

pytestmark = pytest.mark.gpu
P = _native.ptr
BETAS_EPS = (C.c_float(0.9), C.c_float(0.999), C.c_float(1e-5))
LR, MAX_NORM = 2.5e-4, 0.5


def round4(n):
    return (n + 3) // 4 * 4


def payload_words(values):
    """fp64 values -> [len, 4] int32: the words (low half, high half, 0, 0) the kernels store after the gradient."""
    lo_hi = np.asarray(values, dtype=np.float64).view(np.uint32).reshape(-1, 2)
    words = np.concatenate([lo_hi, np.zeros_like(lo_hi)], axis=1).view(np.int32)
    return torch.from_numpy(words.copy())


def rank_order_sum(values):
    s = 0.0
    for v in values:
        s += float(v)
    return s


def f64_bits(x):
    return np.float64(x).view(np.int64)


class KLPeers(up.StagedPeers):
    """StagedPeers that also stage the peers' KL payloads and mirror all W payloads.  kl[parity]: W fp64 values, entry
    `rank` the own one (the mirror of what the kernel stores), or None: no payload in that parity's exchanges."""

    def __init__(self, world, rank, capacity, dev, sliced):
        super().__init__(world, rank, capacity, dev, sliced)
        self.kl = {0: None, 1: None}

    def set_kl(self, values):
        self.kl = {0: values, 1: values}

    def _stage(self, e, peer_grads, n, flag_value):
        staged = super()._stage(e, peer_grads, n, flag_value)
        values = self.kl[e & 1]
        if values is not None:
            words = payload_words(values).to(self.dev)
            off = round4(n)
            for r in range(self.world):
                for buf in ((self.mirror[r],) if r == self.rank else (self.bufs[r], self.mirror[r])):
                    self.slot(buf, e & 1)[off:off + 4].view(torch.int32).copy_(words[r])
        return staged

    def stage_ahead(self, n, steps, peer_grads_by_parity):
        """Before a train() call that makes up to `steps` exchanges: both slots of every peer and every peer flag at the
        last epoch the call can reach.  -> the epoch count before the call."""
        assert int(self.epoch_dev.item()) == self.epoch, 'device epoch out of step with the staging: refusing to stage'
        last = self.epoch + steps
        for parity in (0, 1):
            assert self._stage(parity, peer_grads_by_parity[parity], n, last) == self._polled()
        torch.cuda.synchronize()
        return self.epoch

    def ran(self, exchanges):
        self.epoch += exchanges
        self.check_epoch()

    def close(self):
        pass


# ---- 1. kernels ----------------------------------------------------------------------------------------------------------

WORLDS = [(2, 0), (2, 1), (3, 1), (3, 2), (5, 0), (5, 3), (8, 0), (8, 5), (8, 7)]
# (features, head rows, actions, packed): _DefaultMLPUpdate's buffer, n = 128 F + 1160 (8 head rows) and 128 F + 2192
# (16 head rows) for F = 1, 49, 128; and the six gradients back to back at n = 1411 and 17157 (n % 4 != 0)
SHAPES = [(1, 8, 4, False), (49, 8, 4, False), (128, 8, 4, False), (1, 16, 8, False), (49, 16, 8, False),
          (128, 16, 8, False), (7, 0, 2, True), (128, 0, 4, True)]


def layout(features, rows, n_act, packed):
    hid = 128
    if packed:
        sizes = [hid * features, hid, n_act * hid, n_act, hid, 1]
        return sum(sizes), [(sum(sizes[:i]), sizes[i]) for i in range(6)]
    w_cat, b_enc = hid * features, hid * features + rows * hid
    b_cat = b_enc + hid
    return b_cat + rows, [(0, hid * features), (b_enc, hid), (w_cat, n_act * hid), (b_cat, n_act), (w_cat + n_act * hid, hid),
                          (b_cat + n_act, 1)]


def shape_id(s):
    f, rows, n_act, packed = s
    return f'packed-F{f}-a{n_act}-n{layout(*s)[0]}' if packed else f'F{f}-R{rows}-n{layout(*s)[0]}'


class Engine:
    """One copy of the parameters, Adam state, flat gradient buffer and 8-row head matrix (n_act <= 7: rebuilt by the
    sliced kernel's last CTA)."""

    def __init__(self, params, n, views, n_act, dev):
        self.p = [q.clone() for q in params]
        self.m, self.v = [torch.zeros_like(q) for q in params], [torch.zeros_like(q) for q in params]
        self.step = [torch.zeros((), device=dev) for _ in params]
        self.flat = torch.zeros(n, device=dev)
        self.n = n
        grads = [self.flat[o:o + k] for o, k in views]
        self.arr = (_native.AdamTensor * 6)()
        for i in range(6):
            self.arr[i] = _native.AdamTensor(self.p[i].data_ptr(), self.m[i].data_ptr(), self.v[i].data_ptr(),
                                             self.step[i].data_ptr(), grads[i].data_ptr(), self.p[i].numel())
        self.norm = torch.zeros(1, device=dev)
        self.w_cat, self.b_cat = torch.full((8, 128), 9.0, device=dev), torch.full((8,), 9.0, device=dev)
        self.pack = None if n_act > 7 else _native.HeadPack(
            self.p[2].data_ptr(), self.p[3].data_ptr(), self.p[4].data_ptr(), self.p[5].data_ptr(), self.w_cat.data_ptr(),
            self.b_cat.data_ptr(), n_act, 128)
        self.parts = torch.zeros(up.SLICES, dtype=torch.float64, device=dev)

    def hyper(self, world):
        return (C.c_float(MAX_NORM), C.c_float(1.0 / world), C.c_float(LR), None, *BETAS_EPS, P(self.norm))

    def step_call(self, kernel, world, comm, kl_in=None, kl_out=None, ex=True):
        """One optimizer step with the exchange: kernel 'single' (pb_clip_adam_peer[_ex]) or 'parts' (..._parts[_ex])."""
        lib, s = _native.lib(), _native.stream_ptr()
        if kernel == 'single':
            args = (self.arr, 6, *self.hyper(world), C.byref(comm), P(self.flat), self.n)
            rc = lib.pb_clip_adam_peer_ex(*args, P(kl_in), P(kl_out), s) if ex else lib.pb_clip_adam_peer(*args, s)
        else:
            args = (self.arr, 6, *self.hyper(world), C.byref(comm), P(self.flat), self.n, P(self.parts),
                    C.byref(self.pack) if self.pack is not None else None)
            rc = lib.pb_clip_adam_peer_parts_ex(*args, P(kl_in), P(kl_out), s) if ex else lib.pb_clip_adam_peer_parts(*args, s)
        _native.check(rc)

    def state(self):
        return self.p + self.m + self.v + self.step + [self.norm, self.w_cat, self.b_cat, self.flat]


def default_parameters(features, n_act, dev):
    shapes = [(128, features), (128,), (n_act, 128), (n_act,), (1, 128), (1,)]
    return [torch.randn(s, device=dev) * 0.1 for s in shapes]


def step_gradients(n, views, world, seed, dev, steps=3):
    """Per-rank gradients [W, n], zero outside the six views, mean norm about 0.1; step 1 is 200 times larger (clipped)."""
    mask = torch.zeros(n, device=dev)
    for o, k in views:
        mask[o:o + k] = 1.0
    first = up.gradients(n, world, seed, dev) * mask
    scale = 0.1 / float((first.double().sum(0) / world).norm())
    return [up.gradients(n, world, seed + it, dev, scale * (200.0 if it == 1 else 1.0)) * mask for it in range(steps)]


def kl_values(world, seed):
    """Per-rank payloads of about 1e30 (with a spread, so the fp64 sum's order matters)."""
    gen = np.random.default_rng(seed)
    return [float(v) for v in 1e30 * (1.0 + gen.random(world)) * (1.0 + 1e-9 * gen.standard_normal(world))]


def assert_same(a, b, what):
    names = [f'{k}[{i}]' for k in ('param', 'exp_avg', 'exp_avg_sq', 'step') for i in range(6)] + ['norm', 'w_cat', 'b_cat', 'flat']
    for name, x, y in zip(names, a.state(), b.state()):
        assert torch.equal(up.bits(x), up.bits(y)), f'{what}: {name} differs in {int((up.bits(x) != up.bits(y)).sum())} elements'


@pytest.mark.parametrize('kernel', ['single', 'parts'])
@pytest.mark.parametrize('shape', SHAPES, ids=shape_id)
@pytest.mark.parametrize('world,rank', WORLDS)
def test_ex_kernels_carry_the_kl_sum_beside_an_unchanged_step(world, rank, shape, kernel):
    """Three steps (epochs 1, 2, 3: slots 1, 0, 1) of the _ex kernel with a payload vs the existing entry point without,
    each on its own staged buffers and the same gradients: same bits everywhere but *kl_out; *kl_out is the rank-order
    fp64 sum; every buffer byte as the protocol says (the old kernel's payload floats keep their canaries)."""
    dev = torch.device('cuda')
    torch.manual_seed(17)
    features, _, n_act, _ = shape
    n, views = layout(*shape)
    params = default_parameters(features, n_act, dev)
    ex, old = Engine(params, n, views, n_act, dev), Engine(params, n, views, n_act, dev)
    sliced = kernel == 'parts'
    peers_ex = KLPeers(world, rank, round4(n) + 4, dev, sliced)
    peers_old = KLPeers(world, rank, round4(n) + 4, dev, sliced)
    kl_in = torch.zeros(1, dtype=torch.float64, device=dev)
    kl_out = torch.zeros(1, dtype=torch.float64, device=dev)
    for it, g in enumerate(step_gradients(n, views, world, 31 * n + world, dev)):
        kls = kl_values(world, 1000 * world + 10 * rank + it)
        peers_ex.set_kl(kls)
        kl_in.fill_(kls[rank])
        kl_out.fill_(float('nan'))
        ex.flat.copy_(g[rank])
        old.flat.copy_(g[rank])
        peers_ex.exchange(ex.flat, g, lambda comm: ex.step_call(kernel, world, comm, kl_in, kl_out))
        peers_old.exchange(old.flat, g, lambda comm: old.step_call(kernel, world, comm, ex=False))
        for peers in (peers_ex, peers_old):
            peers.check_epoch()
            peers.check_buffers()
        assert torch.equal(up.bits(ex.flat), up.bits(up.rank_order_sum(g)))
        assert_same(ex, old, f'step {it}, {kernel} with the payload vs without')
        assert float(ex.step[0]) == it + 1
        assert f64_bits(kl_out.item()) == f64_bits(rank_order_sum(kls)), (kl_out.item(), rank_order_sum(kls))


@pytest.mark.parametrize('world,rank,shape', [(2, 1, SHAPES[2]), (8, 0, SHAPES[6]), (5, 3, SHAPES[4])], ids=['2-1', '8-0', '5-3'])
def test_parts_ex_replays_in_a_graph(world, rank, shape):
    """Three pb_clip_adam_peer_parts_ex steps captured in one graph, each carrying its own KL into its own kl_out, replayed
    twice (epochs 1-3 and 4-6) vs the same six steps run eagerly.  Before a replay both slots of every peer are staged, one
    gradient set and one payload set per epoch parity, and every peer flag is set to the last epoch the replay reaches."""
    dev = torch.device('cuda')
    torch.manual_seed(11)
    features, _, n_act, _ = shape
    n, views = layout(*shape)
    params = default_parameters(features, n_act, dev)
    sets = step_gradients(n, views, world, 500 + features, dev, steps=5)
    by_parity = sets[:2]
    kl_by_parity = [kl_values(world, 70 + p) for p in (0, 1)]
    own = [sets[3][0], sets[1][0], sets[4][0]]
    own_kl = torch.tensor([3e29, float('inf'), 5e29], dtype=torch.float64, device=dev)

    def peer_kls(parity, it):
        v = list(kl_by_parity[parity])
        v[rank] = float(own_kl[it % 3])
        return v

    eager, graphed = Engine(params, n, views, n_act, dev), Engine(params, n, views, n_act, dev)
    out_e = torch.zeros(3, dtype=torch.float64, device=dev)
    out_g = torch.zeros(3, dtype=torch.float64, device=dev)
    peers_e = KLPeers(world, rank, round4(n) + 4, dev, sliced=True)
    after = []
    for it in range(6):
        parity = (it + 1) & 1
        peers_e.set_kl(peer_kls(parity, it))
        eager.flat.copy_(own[it % 3])
        peers_e.exchange(eager.flat, by_parity[parity],
                         lambda comm: eager.step_call('parts', world, comm, own_kl[it % 3:it % 3 + 1], out_e[it % 3:it % 3 + 1]))
        if it % 3 == 2:
            after.append([t.clone() for t in eager.state()] + [out_e.clone()])
    peers_e.check_epoch()

    def three_steps(comm):
        for it in range(3):
            graphed.flat.copy_(own[it])
            graphed.step_call('parts', world, comm, own_kl[it:it + 1], out_g[it:it + 1])

    peers_g = KLPeers(world, rank, round4(n) + 4, dev, sliced=True)
    graph = peers_g.capture(three_steps)
    for replay in range(2):
        # epochs 3 r + 1 .. 3 r + 3 have parities (1, 0, 1) then (0, 1, 0): the own payload differs per step, the staged
        # peer payloads per parity; a parity's own entry only feeds the mirror, which a replay does not check
        peers_g.kl = {p: kl_by_parity[p] for p in (0, 1)}
        out_g.fill_(float('nan'))
        peers_g.replay(graph, by_parity, n, 3)
        torch.cuda.synchronize()
        peers_g.check_epoch()
        for i, (x, y) in enumerate(zip([t for t in graphed.state()] + [out_g], after[replay])):
            assert torch.equal(up.bits(x) if x.dtype == torch.float32 else x.view(torch.int64),
                               up.bits(y) if y.dtype == torch.float32 else y.view(torch.int64)), (replay, i)
        for it in range(3):
            parity = (3 * replay + it + 1) & 1
            assert f64_bits(out_g[it].item()) == f64_bits(rank_order_sum(peer_kls(parity, it))), (replay, it)


def test_ex_argument_checks():
    """Refused on the host, nothing launched: no room for the payload, one of kl_in / kl_out alone, a misaligned kl_in or
    kl_out, a payload without a communicator of 2 or more ranks.  Every flag is far ahead of the epoch, so a check that
    stopped firing would run through instead of waiting."""
    dev = torch.device('cuda')
    lib, s = _native.lib(), _native.stream_ptr()
    peers = KLPeers(8, 0, 64, dev, sliced=True)
    for buf in peers.bufs:
        buf[:up.HEADER_WORDS] = 1 << 40
    n, views = 16, [(0, 4), (4, 4), (8, 2), (10, 2), (12, 2), (14, 2)]
    eng = Engine([torch.zeros(k, device=dev) for _, k in views], n, views, 2, dev)
    kl = torch.zeros(4, dtype=torch.float64, device=dev)
    kl_in, kl_out = kl[0:1], kl[1:2]
    odd = C.c_void_p(kl.data_ptr() + 4)

    def comm(**changes):
        c = _native.PeerComm.from_buffer_copy(peers.struct)
        for k, v in changes.items():
            setattr(c, k, v)
        return c

    fits, tight = comm(capacity=20), comm(capacity=19)
    hyper = eng.hyper(8)
    bad = [('no room', tight, P(kl_in), P(kl_out)), ('kl_in alone', fits, P(kl_in), None),
           ('kl_out alone', fits, None, P(kl_out)), ('misaligned kl_in', fits, odd, P(kl_out)),
           ('misaligned kl_out', fits, P(kl_in), odd), ('world 1', comm(capacity=20, world=1), P(kl_in), P(kl_out))]
    launches = lib.pb_launch_count()
    for what, c, a, b in bad:
        calls = {
            'pb_clip_adam_peer_ex': lambda: lib.pb_clip_adam_peer_ex(eng.arr, 6, *hyper, C.byref(c), P(eng.flat), n, a, b, s),
            'pb_clip_adam_peer_parts_ex': lambda: lib.pb_clip_adam_peer_parts_ex(
                eng.arr, 6, *hyper, C.byref(c), P(eng.flat), n, P(eng.parts), None, a, b, s),
        }
        for name, call in calls.items():
            with pytest.raises(APIUsageError, match=f'^{name}: '):
                _native.check(call())
            assert lib.pb_launch_count() == launches, (what, name)
    with pytest.raises(APIUsageError, match='^pb_clip_adam_peer_ex: a KL payload needs'):
        _native.check(lib.pb_clip_adam_peer_ex(eng.arr, 6, *hyper, None, P(eng.flat), n, P(kl_in), P(kl_out), s))
    assert lib.pb_launch_count() == launches
    peers.check_epoch()


# ---- 2. the decision -----------------------------------------------------------------------------------------------------

M = 4096                     # rows per minibatch on every rank
T = 0.02


def decision_cases(world):
    """name -> (function own rank -> W fp64 KL row sums, target_kl values, decisions expected for them).  Row sums are
    M times a mean approx_kl."""
    gen = np.random.default_rng(world)
    fixed = [float(x) for x in gen.random(world) * 0.04 * M]
    v = np.float32(np.float64(rank_order_sum(fixed)) / (world * M))
    near = [float(np.nextafter(v, np.float32(-np.inf))), float(v), float(np.nextafter(v, np.float32(np.inf)))]
    nan = [0.5 * T * M] * (world - 1) + [float('nan')]
    inf = [0.1 * T * M] * (world - 1) + [float('inf')]
    return {
        # this rank alone would stop (1.5 T), the mean over the ranks is below T
        'own_above_mean_below': (lambda k: [1.5 * T * M if r == k else 0.1 * T * M for r in range(world)], [T], [False]),
        # this rank alone would go on (0.5 T), the mean is above T
        'own_below_mean_above': (lambda k: [0.5 * T * M if r == k else 2.0 * T * M for r in range(world)], [T], [True]),
        # the same sums at every position; targets at fp32(mean) and one ulp either side
        'fp32_neighbours': (lambda k: fixed, near, [True, False, False]),
        'nan_on_one_rank': (lambda k: nan, [T, 0.0], [False, False]),
        'inf_on_one_rank': (lambda k: inf, [T, 1e30], [True, True]),
    }


@pytest.mark.parametrize('case', ['own_above_mean_below', 'own_below_mean_above', 'fp32_neighbours', 'nan_on_one_rank',
                                  'inf_on_one_rank'])
@pytest.mark.parametrize('world', [2, 3, 8])
def test_one_decision_at_every_rank_position(world, case):
    """For each own-rank position k: an exchange of pb_clip_adam_peer_parts_ex carrying the sums, then pb_kl_stop on
    *kl_out with rows = W * M.  The decision is the rule's at every position; where the sums do not depend on k, *kl_out
    has the same bits at every position."""
    dev = torch.device('cuda')
    torch.manual_seed(3)
    shape = SHAPES[6]
    n, views = layout(*shape)
    params = default_parameters(shape[0], shape[2], dev)
    sums_of, targets, want = decision_cases(world)[case]
    tgt = torch.tensor(targets, dtype=torch.float32, device=dev)
    g = step_gradients(n, views, world, 9, dev, steps=1)[0]
    kl_in = torch.zeros(1, dtype=torch.float64, device=dev)
    kl_out = torch.zeros(1, dtype=torch.float64, device=dev)
    state = torch.zeros(2, dtype=torch.int32, device=dev)
    outs = []
    for k in range(world):
        sums = sums_of(k)
        eng = Engine(params, n, views, shape[2], dev)
        peers = KLPeers(world, k, round4(n) + 4, dev, sliced=True)
        peers.set_kl(sums)
        kl_in.fill_(sums[k])
        eng.flat.copy_(g[k])
        peers.exchange(eng.flat, g, lambda comm: eng.step_call('parts', world, comm, kl_in, kl_out))
        peers.check_buffers()
        total = rank_order_sum(sums)
        if np.isnan(total):             # the device's NaN need not carry the payload bits of the staged one
            assert np.isnan(kl_out.item()), (k, kl_out.item())
        else:
            assert f64_bits(kl_out.item()) == f64_bits(total), (k, kl_out.item(), total)
        outs.append(f64_bits(kl_out.item()))
        got = []
        for i in range(len(targets)):
            _native.check(_native.lib().pb_kl_stop(None, P(kl_out), world * M, P(tgt[i:i + 1]), 0, P(state), 0, 0,
                                                   _native.stream_ptr()))
            got.append(bool(state[0].item()))
        rule = [bool(np.float32(np.float64(total) / (world * M)) > np.float32(t)) for t in targets]
        assert got == rule == want, (case, k, got, rule, want)
    if case in ('fp32_neighbours', 'nan_on_one_rank', 'inf_on_one_rank'):
        assert len(set(outs)) == 1, outs


# ---- 3. train() playing rank k of 2 --------------------------------------------------------------------------------------

# name -> (env, num_envs, horizon, config overrides, engine, sliced exchange)
PLANS = {
    'mlp_fused': ('breakout', 64, 128, {}, 'mlp_fused', True),
    'mlp_chain_squared': ('squared', 64, 32, dict(bptt_horizon=8), 'mlp_chain', False),
}
WORLD = 2


def adam_state(opt):
    return [opt.state[p][k] for p in opt.param_groups[0]['params'] for k in ('exp_avg', 'exp_avg_sq', 'step')]


def as_ranks(monkeypatch, rank, sliced, nflat, made):
    """torch.distributed as seen by rank `rank` of 2, with no process group (the only collective train() makes on the
    peer plan is the agreement on PeerComm, which finds every rank agreeing); distributed.PeerComm -> KLPeers, staged for
    the first train() call as it is made, before the trainer can launch an exchange."""
    import torch.distributed as dist
    import pufferlib_b200.distributed as pdist
    monkeypatch.setattr(dist, 'is_initialized', lambda: True)
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: WORLD)
    monkeypatch.setattr(dist, 'get_rank', lambda group=None: rank)
    monkeypatch.setattr(dist, 'all_reduce', lambda tensor, op=None, group=None, async_op=False: None)

    def staged(capacity):
        assert capacity == round4(nflat) + 4, 'the peer slot must have room for the KL payload'
        peers = KLPeers(WORLD, rank, capacity, torch.device('cuda'), sliced=sliced)
        peers.set_kl([0.0] * WORLD)
        zero = torch.zeros(WORLD, nflat, device='cuda')
        peers.stage_ahead(nflat, 3, [zero, zero])
        made.append(peers)
        return peers
    monkeypatch.setattr(pdist, 'PeerComm', staged)


def snapshot(data, pol):
    return [p.detach().clone() for p in pol.parameters()], [t.clone() for t in adam_state(data.optimizer)]


def restore(data, pol, snap):
    with torch.no_grad():
        for p, s in zip(pol.parameters(), snap[0]):
            p.copy_(s)
        for t, s in zip(adam_state(data.optimizer), snap[1]):
            t.copy_(s)
    clean_pufferl._invalidate_policy_cache(data)


@pytest.mark.parametrize('rank', [0, 1])
@pytest.mark.parametrize('name', list(PLANS))
def test_train_stops_as_the_mean_over_the_ranks_decides(name, rank, monkeypatch):
    env, n, h, kw, engine, sliced = PLANS[name]
    made = []
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=7).cuda()
    (n_act, hid), features = pol.policy.decoder.weight.shape, pol.policy.encoder.weight.shape[1]
    rows = next(r for r in (8, 16, 32) if n_act + 1 <= r)
    nflat = hid * features + rows * hid + hid + rows        # _DefaultMLPUpdate's flat gradient buffer
    as_ranks(monkeypatch, rank, sliced, nflat, made)
    cfg = dict(seed=1, torch_deterministic=True, env=env, batch_size=n * h, bptt_horizon=16, minibatch_size=n * h,
               cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
               update_epochs=3, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5,
               ent_coef=0.01, max_grad_norm=0.5, target_kl=1e9, anneal_lr=False, total_timesteps=10 ** 9, cuda_graph=True)
    cfg.update(kw)
    data = clean_pufferl.create(clean_pufferl.pufferlib_b200.namespace(**cfg), vec, pol)
    assert data.grad_bucket is not None and data.experience.num_minibatches == 1

    def run(peer_sum, captured):
        """One train() with the peer's KL row sum staged for every exchange (zero peer gradients) -> epochs run.  The
        first call's staging is made by the communicator's factory."""
        if made:
            zero = torch.zeros(WORLD, nflat, device='cuda')
            made[0].set_kl([peer_sum] * WORLD)
            before = made[0].stage_ahead(nflat, 3, [zero, zero])
        else:
            assert peer_sum == 0.0
            before = 0
        data.config.cuda_graph_train = captured
        r0 = data.train_graph_replays
        clean_pufferl.train(data)
        torch.cuda.synchronize()
        peers = made[0]
        peers.ran(data.train_epochs_run)          # one minibatch per epoch: one exchange per epoch that ran
        assert peers.epoch == before + data.train_epochs_run
        if captured and data.train_graph_state == 2 and r0 > 0:
            assert data.train_graph_replays == r0 + 1
        return data.train_epochs_run

    clean_pufferl.evaluate(data)
    assert run(0.0, True) == 3                    # eager first call (initialises Adam)
    assert len(made) == 1 and data.manual_update.gflat.numel() == nflat and data.manual_update.peer is made[0]
    clean_pufferl.evaluate(data)
    assert run(0.0, True) == 3                    # capture + first replay
    assert data.train_graph_state == 2, data.msg
    plan = clean_pufferl.update_plan(data)
    assert (plan.engine, plan.capture) == (engine, 'whole'), plan

    clean_pufferl.evaluate(data)
    snap = snapshot(data, pol)
    run(0.0, False)                               # probe: this rank's KL row sums of epochs 0 and 1
    mb_rows = data.manual_update.mb_rows
    sums = [float(data.manual_update.stats[e, 4]) for e in (0, 1)]
    own = [s / mb_rows for s in sums]        # epoch 0's may be exactly 0: its parameters are the rollout's
    assert max(own) > 0, own

    def rule(peer_sum, target):
        for e in (0, 1):
            total = rank_order_sum([sums[e], peer_sum] if rank == 0 else [peer_sum, sums[e]])
            v = np.float32(np.float64(total) / (WORLD * mb_rows))
            assert abs(float(v) - np.float32(target)) > 1e-3 * target, 'a decision too close to call'
            if v > np.float32(target):
                return e + 1
        return 3

    def alone(target):
        return next((e + 1 for e in (0, 1) if np.float32(own[e]) > np.float32(target)), 3)

    t_up = 1.5 * max(own)                         # alone: never stops; the peer's large KL makes the mean stop
    t_down = 0.75 * max(own)                      # alone: stops after epoch 0 or 1; the peer's zero KL halves the mean
    cases = [(t_up, 4.0 * t_up * mb_rows), (t_down, 0.0)]
    for target, peer_sum in cases:
        want = rule(peer_sum, target)
        assert want != alone(target), (target, want, alone(target))
        data.config.target_kl = target
        restore(data, pol, snap)
        ep_e = run(peer_sum, False)
        ref = snapshot(data, pol)
        restore(data, pol, snap)
        launches = _native.lib().pb_launch_count()
        ep_c = run(peer_sum, True)
        assert _native.lib().pb_launch_count() == launches and data.train_graph_state == 2
        got = snapshot(data, pol)
        print(f'[target_kl ranks] {name} rank {rank}: target {target:.4g}, peer sum {peer_sum:.4g}: epochs eager {ep_e} '
              f'captured {ep_c}, own alone {alone(target)}; params bitwise '
              f'{all(torch.equal(a, b) for a, b in zip(got[0], ref[0]))}', flush=True)
        assert ep_e == ep_c == want, (target, ep_e, ep_c, want)
        for what, a_list, b_list in (('params', got[0], ref[0]), ('adam', got[1], ref[1])):
            for i, (a, b) in enumerate(zip(a_list, b_list)):
                assert torch.equal(a, b), (what, i, float((a - b).abs().max()))
        assert float(adam_state(data.optimizer)[2]) - float(snap[1][2]) == want
    clean_pufferl.close(data)
