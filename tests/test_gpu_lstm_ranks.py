"""The recurrent update on several ranks, on ONE device against staged peers (tests/util_peer.py): the gradient mean over NVLink
peer memory (pb_peer_allreduce_mean, csrc/peer.cu) and train() with RecurrentPolicy(LSTMWrapper(Default), fused_update=True)
playing rank k of 2, its whole update captured in one CUDA graph.

1. ABI.  Every bad argument is refused on the host: nothing launched, no byte of any buffer changed.
2. Arithmetic.  At the LSTM's flat gradient sizes and at every own-rank position of worlds 2, 3, 4 and 8 (and one of 5, 6,
   7, where 1/world is inexact), the result is bitwise the fp32 rank-order sum times fp32(1/world), which is what
   GradBucket.all_reduce_mean's torch.div_ gives for that sum; the payload is bitwise the rank-order fp64 sum; every byte of
   all W buffers is as the protocol says and the epoch advances by one per call -- eager, and in a graph replayed 3 times.
3. train() as rank k of 2: plan ('bptt', 'segments', 'whole'), a replay that launches nothing from the host, captured equal
   to eager bitwise, and the peer plan equal to the NCCL plan bitwise.
4. target_kl: the epochs run, captured and eager, are the ones the KL mean over both ranks decides.

No test here lets a kernel wait: every launch that polls flags is staged first (StagedPeers.exchange / replay, or
KLPeers.stage_ahead before a train() call, which stages every exchange the call can make).
"""
import ctypes as C

import numpy as np
import pytest
import torch

from pufferlib_b200 import _native, clean_pufferl
from pufferlib_b200.exceptions import APIUsageError

import util_peer as up
from test_gpu_lstm_train_graph import make_recurrent
from test_gpu_policy_lstm import make_config
from test_gpu_target_kl_ranks import (KLPeers, adam_state, as_ranks, f64_bits, kl_values, payload_words, rank_order_sum,
                                      restore, round4, snapshot)

pytestmark = pytest.mark.gpu
P = _native.ptr


def lstm_flat(hidden, features, n_act):
    """GradBucket's size for LSTMWrapper(Default): encoder, decoder, value head, then the LSTM's four tensors."""
    return hidden * features + hidden + (hidden + 1) * n_act + hidden + 1 + 2 * 4 * hidden * hidden + 2 * 4 * hidden


assert lstm_flat(128, 128, 4) == 149253 and lstm_flat(256, 128, 4) == 560645

# H = 128 with F in {1, 49, 128} and 2 / 4 / 15 actions, H = 256 with F = 128; then n % 4 != 0 below 900, where the trailing
# slices of the 16-slice exchange are empty
SIZES = [lstm_flat(128, f, a) for f in (1, 49, 128) for a in (2, 4, 15)] + [lstm_flat(256, 128, 4), 5, 899]
WORLDS = [(w, k) for w in (2, 3, 4, 8) for k in range(w)] + [(5, 2), (6, 5), (7, 0)]


def mean_call(flat, kl_in=None, kl_out=None):
    lib, s = _native.lib(), _native.stream_ptr()
    return lambda comm: _native.check(lib.pb_peer_allreduce_mean(C.byref(comm), P(flat), flat.numel(), P(kl_in), P(kl_out), s))


def expected_mean(g):
    """GradBucket.all_reduce_mean on the rank-order sum: torch's flat.div_(world) on the device."""
    s = up.rank_order_sum(g)
    return s.div_(g.shape[0])


# ---- 1. argument checks --------------------------------------------------------------------------------------------------

def test_mean_argument_checks():
    """Refused before any launch, with every flag of every buffer far ahead of the epoch (a check that stopped firing would
    run through rather than wait): the communicator checks of pb_peer_allreduce_parts, and the payload's (one of kl_in /
    kl_out alone, misaligned, no room after round4(n), fewer than 2 ranks).  Launch count and every byte unchanged."""
    dev = torch.device('cuda')
    lib, s = _native.lib(), _native.stream_ptr()
    peers = KLPeers(8, 0, 64, dev, sliced=True)
    for buf in peers.bufs:
        buf[:up.HEADER_WORDS] = 1 << 40
    n = 16
    flat = torch.arange(n, dtype=torch.float32, device=dev)
    kl = torch.tensor([1.5, 2.5, 3.5, 4.5], dtype=torch.float64, device=dev)
    kl_in, kl_out, odd = P(kl[0:1]), P(kl[1:2]), C.c_void_p(kl.data_ptr() + 4)

    def comm(**changes):
        c = _native.PeerComm.from_buffer_copy(peers.struct)
        for key, value in changes.items():
            if key.startswith('base'):
                c.base[int(key[4:])] = value
            else:
                setattr(c, key, value)
        return c

    before = [t.clone() for t in peers.bufs + [flat, kl, peers.epoch_dev]]
    bad = [('world = 9', comm(capacity=20, world=9), P(flat), n, None, None),
           ('world = 0', comm(capacity=20, world=0, rank=0), P(flat), n, None, None),
           ('rank = world', comm(capacity=20, rank=8), P(flat), n, None, None),
           ('negative rank', comm(capacity=20, rank=-1), P(flat), n, None, None),
           ('n > capacity', comm(capacity=15), P(flat), n, None, None),
           ('n = 0', comm(capacity=20), P(flat), 0, None, None),
           ('null flat', comm(capacity=20), None, n, None, None),
           ('null base', comm(capacity=20, base5=None), P(flat), n, None, None),
           ('null epoch', comm(capacity=20, epoch=None), P(flat), n, None, None),
           ('no room for the payload', comm(capacity=19), P(flat), n, kl_in, kl_out),
           ('kl_in alone', comm(capacity=20), P(flat), n, kl_in, None),
           ('kl_out alone', comm(capacity=20), P(flat), n, None, kl_out),
           ('misaligned kl_in', comm(capacity=20), P(flat), n, odd, kl_out),
           ('misaligned kl_out', comm(capacity=20), P(flat), n, kl_in, odd),
           ('payload on one rank', comm(capacity=20, world=1), P(flat), n, kl_in, kl_out)]
    launches = lib.pb_launch_count()
    for what, c, f, count, a, b in bad:
        with pytest.raises(APIUsageError, match='^pb_peer_allreduce_mean: '):
            _native.check(lib.pb_peer_allreduce_mean(C.byref(c), f, count, a, b, s))
        assert lib.pb_launch_count() == launches, what
    with pytest.raises(APIUsageError, match='^pb_peer_allreduce_mean: '):
        _native.check(lib.pb_peer_allreduce_mean(None, P(flat), n, None, None, s))
    assert lib.pb_launch_count() == launches
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(peers.bufs + [flat, kl, peers.epoch_dev], before)):
        assert torch.equal(x, y), f'tensor {i} changed by a refused call'


# ---- 2. arithmetic -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('n', SIZES)
@pytest.mark.parametrize('world,rank', WORLDS)
def test_mean_is_the_rank_order_sum_scaled_like_grad_bucket(world, rank, n):
    """Three calls (epochs 1, 2, 3: slots 1, 0, 1), the first and last carrying a payload of about 1e30, the middle one none
    (its payload floats keep what the slot held).  capacity = round4(n) + 4, the trainer's."""
    dev = torch.device('cuda')
    peers = KLPeers(world, rank, round4(n) + 4, dev, sliced=True)
    flat = torch.zeros(n, device=dev)
    kl_in = torch.zeros(1, dtype=torch.float64, device=dev)
    kl_out = torch.zeros(1, dtype=torch.float64, device=dev)
    for call in range(3):
        g = up.gradients(n, world, 7 * n + 100 * world + 10 * rank + call, dev)
        flat.copy_(g[rank])
        if call == 1:
            peers.kl = {0: None, 1: None}
            launch = mean_call(flat)
        else:
            kls = kl_values(world, 1000 * world + 10 * rank + call)
            peers.set_kl(kls)
            kl_in.fill_(kls[rank])
            kl_out.fill_(float('nan'))
            launch = mean_call(flat, kl_in, kl_out)
        assert peers.exchange(flat, g, launch) == call + 1
        peers.check_epoch()
        peers.check_buffers()
        want = expected_mean(g)
        assert torch.equal(up.bits(flat), up.bits(want)), \
            f'{int((up.bits(flat) != up.bits(want)).sum())} of {n} elements differ from the rank-order sum / {world}'
        if call != 1:
            assert f64_bits(kl_out.item()) == f64_bits(rank_order_sum(kls)), (kl_out.item(), rank_order_sum(kls))
        if world in (3, 5, 6, 7) and n > 1000:
            # the test tells the reciprocal from a true division: at these worlds the two differ somewhere
            quotient = (up.rank_order_sum(g).double() / world).float()
            assert not torch.equal(up.bits(flat), up.bits(quotient))


def own_writes(peers, e, own, own_kl, n):
    """The mirror of what the own rank's call of epoch e leaves: its gradient in its slot, its payload after it (or
    nothing), its 16 slice flags = e in every buffer."""
    k = peers.rank
    slot = peers.slot(peers.mirror[k], e & 1)
    slot[:n].copy_(own)
    if own_kl is not None:
        slot[round4(n):round4(n) + 4].view(torch.int32).copy_(payload_words([own_kl])[0].to(peers.dev))
    for r in range(peers.world):
        peers.mirror[r][torch.tensor([16 * k + b for b in range(up.SLICES)], device=peers.dev)] = e


@pytest.mark.parametrize('world,rank,n', [(2, 1, lstm_flat(128, 128, 4)), (3, 0, lstm_flat(256, 128, 4)), (8, 5, 899),
                                          (4, 2, lstm_flat(128, 1, 2))])
def test_mean_replays_in_a_graph(world, rank, n):
    """Three calls captured in one graph, each on its own input and with its own payload, replayed 3 times: every call's
    result and payload sum bitwise as the rule says, the epoch advanced by 3 per replay, every buffer byte as the protocol
    says after each replay.  Both slots of every peer are staged, one gradient and payload set per parity."""
    dev = torch.device('cuda')
    by_parity = [up.gradients(n, world, 40 + p, dev) for p in (0, 1)]
    kl_by_parity = [kl_values(world, 70 + p) for p in (0, 1)]
    own = up.gradients(n, 3, 90, dev)
    own_kl = torch.tensor([3e29, 7e29, -5e29], dtype=torch.float64, device=dev)
    flat = torch.zeros(n, device=dev)
    outs = torch.zeros(3, n, device=dev)
    kl_out = torch.zeros(3, dtype=torch.float64, device=dev)
    peers = KLPeers(world, rank, round4(n) + 4, dev, sliced=True)
    peers.kl = {p: kl_by_parity[p] for p in (0, 1)}

    def three_calls(comm):
        lib, s = _native.lib(), _native.stream_ptr()
        for i in range(3):
            flat.copy_(own[i])
            _native.check(lib.pb_peer_allreduce_mean(C.byref(comm), P(flat), n, P(own_kl[i:i + 1]), P(kl_out[i:i + 1]), s))
            outs[i].copy_(flat)

    graph = peers.capture(three_calls)
    for replay in range(3):
        outs.fill_(float('nan'))
        kl_out.fill_(float('nan'))
        first = peers.epoch + 1
        peers.replay(graph, by_parity, n, 3)
        torch.cuda.synchronize()
        peers.check_epoch()
        assert peers.epoch == 3 * (replay + 1)
        for i in range(3):
            e = first + i
            g = by_parity[e & 1].clone()
            g[rank] = own[i]
            assert torch.equal(up.bits(outs[i]), up.bits(expected_mean(g))), (replay, i)
            kls = list(kl_by_parity[e & 1])
            kls[rank] = float(own_kl[i])
            assert f64_bits(kl_out[i].item()) == f64_bits(rank_order_sum(kls)), (replay, i)
            own_writes(peers, e, own[i], float(own_kl[i]), n)
        peers.check_buffers()


# ---- 3. train() playing rank k of 2 --------------------------------------------------------------------------------------

# name -> (env, num_envs, horizon, bptt horizon, hidden)
CASES = {
    'breakout': ('breakout', 64, 64, 16, 128),
    'squared': ('squared', 64, 32, 8, 128),
    'memory': ('memory', 64, 32, 8, 128),
    'breakout_h256': ('breakout', 64, 64, 16, 256),
}
WORLD = 2


def recurrent_trainer(name, rank, monkeypatch, made, **kw):
    """RecurrentPolicy(LSTMWrapper(Default), fused_sample=True, fused_update=True) as rank `rank` of 2, one minibatch per
    epoch (so one exchange per epoch), with distributed.PeerComm replaced by staged peers.  -> (data, policy, flat size)."""
    env, n, h, bptt, hidden = CASES[name]
    vec, net, pol = make_recurrent(env, n, hidden=hidden)
    nflat = sum(p.numel() for p in pol.parameters() if p.requires_grad)
    as_ranks(monkeypatch, rank, True, nflat, made)
    cfg = make_config(n, h, env=env, bptt_horizon=bptt, minibatch_size=n * h, cuda_graph=True, **kw)
    data = clean_pufferl.create(cfg, vec, pol)
    assert data.grad_bucket is not None and data.grad_bucket.flat.numel() == nflat
    assert data.experience.num_minibatches == 1
    return data, pol, nflat


def peer_gradient(nflat, rank):
    """The other rank's gradient, the same in both parities: small, mixed signs (row `rank` unused)."""
    g = up.gradients(nflat, WORLD, 5 + nflat, 'cuda', scale=1e-4)
    return [g, g]


@pytest.mark.parametrize('rank', [0, 1])
@pytest.mark.parametrize('name', list(CASES))
def test_train_captures_the_whole_update_and_matches_eager_and_nccl(name, rank, monkeypatch):
    made = []
    data, pol, nflat = recurrent_trainer(name, rank, monkeypatch, made)
    epochs = data.config.update_epochs
    peer_g = peer_gradient(nflat, rank)

    def run(captured):
        """One train() with the peer gradient staged for every exchange -> exchanges made."""
        if made:
            made[0].stage_ahead(nflat, epochs, peer_g)
        data.config.cuda_graph_train = captured
        clean_pufferl.train(data)
        torch.cuda.synchronize()
        made[0].ran(epochs)                        # one minibatch per epoch: one exchange per epoch

    clean_pufferl.evaluate(data)
    run(True)                                      # eager first call (initialises Adam, opens the communicator)
    assert len(made) == 1 and data.grad_bucket.peer is made[0]
    clean_pufferl.evaluate(data)
    run(True)                                      # capture + first replay
    assert data.train_graph_state == 2, data.msg
    plan = clean_pufferl.update_plan(data)
    assert (plan.engine, plan.form, plan.capture) == ('bptt', 'segments', 'whole'), plan
    assert plan.bptt_peer and data.train_recurrent_path == 'fused'

    clean_pufferl.evaluate(data)
    snap = snapshot(data, pol)
    launches, replays = _native.lib().pb_launch_count(), data.train_graph_replays
    run(True)
    assert _native.lib().pb_launch_count() == launches and data.train_graph_replays == replays + 1
    got = snapshot(data, pol)

    restore(data, pol, snap)
    run(False)
    ref = snapshot(data, pol)
    for what, a_list, b_list in (('params', got[0], ref[0]), ('adam', got[1], ref[1])):
        for i, (a, b) in enumerate(zip(a_list, b_list)):
            assert torch.equal(a, b), (f'captured vs eager: {what}', i, float((a - b).abs().max()))

    # the NCCL plan: all_reduce adds the other rank's gradient (x + y == y + x: the rank order does not change the bits),
    # then GradBucket.all_reduce_mean divides by the world
    import torch.distributed as dist
    flat = data.grad_bucket.flat
    calls = []

    def nccl_sum(tensor, op=None, group=None, async_op=False):
        assert tensor.data_ptr() == flat.data_ptr(), 'the NCCL plan makes no other collective here'
        tensor.add_(peer_g[0][1 - rank])
        calls.append(1)
    monkeypatch.setattr(dist, 'all_reduce', nccl_sum)
    data.grad_bucket.close_peer()
    data.config.peer_allreduce = False
    restore(data, pol, snap)
    data.config.cuda_graph_train = False
    clean_pufferl.train(data)
    plan = clean_pufferl.update_plan(data)
    assert not plan.bptt_peer and plan.capture is None and data.grad_bucket.peer is None
    assert len(calls) == epochs
    nccl = snapshot(data, pol)
    print(f'[lstm ranks] {name} rank {rank}: n = {nflat}, captured == eager == NCCL plan, bitwise', flush=True)
    for what, a_list, b_list in (('params', nccl[0], ref[0]), ('adam', nccl[1], ref[1])):
        for i, (a, b) in enumerate(zip(a_list, b_list)):
            assert torch.equal(a, b), (f'NCCL plan vs peer plan: {what}', i, float((a - b).abs().max()))
    clean_pufferl.close(data)


# ---- 4. target_kl --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('rank', [0, 1])
@pytest.mark.parametrize('name', ['breakout', 'squared'])
def test_train_stops_as_the_mean_over_the_ranks_decides(name, rank, monkeypatch):
    """test_gpu_target_kl_ranks.py's test of the same name on the 'bptt' engine: the peer's KL row sum is staged as the
    payload of every exchange, and the epochs run, eager and captured, are those the fp64 rule on the sum over both ranks
    gives, not those this rank alone would stop after; captured equal to eager bitwise."""
    made = []
    data, pol, nflat = recurrent_trainer(name, rank, monkeypatch, made, update_epochs=3, target_kl=1e9)
    rows = data.experience.minibatch_size
    zero = torch.zeros(WORLD, nflat, device='cuda')

    def run(peer_sum, captured):
        if made:
            made[0].set_kl([peer_sum] * WORLD)
            before = made[0].stage_ahead(nflat, 3, [zero, zero])
        else:
            assert peer_sum == 0.0
            before = 0
        data.config.cuda_graph_train = captured
        clean_pufferl.train(data)
        torch.cuda.synchronize()
        made[0].ran(data.train_epochs_run)
        assert made[0].epoch == before + data.train_epochs_run
        return data.train_epochs_run

    clean_pufferl.evaluate(data)
    assert run(0.0, True) == 3
    clean_pufferl.evaluate(data)
    assert run(0.0, True) == 3
    assert data.train_graph_state == 2, data.msg
    plan = clean_pufferl.update_plan(data)
    assert (plan.engine, plan.capture) == ('bptt', 'whole'), plan

    # probe: this rank's KL row sums of epochs 0 and 1, as the exchange carries them
    import pufferlib_b200.distributed as pdist
    seen = []
    real = pdist.GradBucket.peer_all_reduce_mean

    def record(self, kl_in=None, kl_out=None):
        if kl_in is not None:
            seen.append(float(kl_in))
        return real(self, kl_in, kl_out)
    clean_pufferl.evaluate(data)
    snap = snapshot(data, pol)
    monkeypatch.setattr(pdist.GradBucket, 'peer_all_reduce_mean', record)
    assert run(0.0, False) == 3
    monkeypatch.setattr(pdist.GradBucket, 'peer_all_reduce_mean', real)
    assert len(seen) == 2, seen
    own = [s / rows for s in seen]
    assert max(own) > 0, own

    def rule(peer_sum, target):
        for e in (0, 1):
            total = rank_order_sum([seen[e], peer_sum] if rank == 0 else [peer_sum, seen[e]])
            v = np.float32(np.float64(total) / (WORLD * rows))
            assert abs(float(v) - np.float32(target)) > 1e-3 * target, 'a decision too close to call'
            if v > np.float32(target):
                return e + 1
        return 3

    def alone(target):
        return next((e + 1 for e in (0, 1) if np.float32(own[e]) > np.float32(target)), 3)

    t_up = 1.5 * max(own)                         # alone: never stops; the peer's large KL makes the mean stop
    t_down = 0.75 * max(own)                      # alone: stops after epoch 0 or 1; the peer's zero KL halves the mean
    for target, peer_sum in [(t_up, 4.0 * t_up * rows), (t_down, 0.0)]:
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
        print(f'[target_kl lstm ranks] {name} rank {rank}: target {target:.4g}, peer sum {peer_sum:.4g}: epochs eager {ep_e} '
              f'captured {ep_c}, own alone {alone(target)}', flush=True)
        assert ep_e == ep_c == want, (target, ep_e, ep_c, want)
        for what, a_list, b_list in (('params', got[0], ref[0]), ('adam', got[1], ref[1])):
            for i, (a, b) in enumerate(zip(a_list, b_list)):
                assert torch.equal(a, b), (what, i, float((a - b).abs().max()))
        assert float(adam_state(data.optimizer)[2]) - float(snap[1][2]) == want
    clean_pufferl.close(data)
