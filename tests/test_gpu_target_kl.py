"""target_kl decided on the device (reference clean_pufferl.py:256-258: after each epoch, `if approx_kl > target_kl: break`
on the last minibatch's approx_kl).

1. pb_kl_stop alone (csrc/graph_cond.cu): every decision equals torch's `bool(torch.tensor(a) > t)` at fp32(t) and one
   ulp either side, at NaN and +-inf, from an fp32 scalar and from an fp64 statistics row (whose fp32 value is bitwise
   fused_ppo_loss's approx_kl for the same rows).
2. The IF-node helpers alone: one captured graph with four IF bodies gated by pb_kl_stop, replayed so that 1 to 4 bodies
   run; every handle is back at its default at the start of a replay and was created on the root graph; the helpers
   refuse to run outside a capture.
3. train() with target_kl, captured, on four engine / minibatch-form plans (the hand-written update fused and as a
   kernel chain, autograd on the packed heads, the BPTT kernels), against eager train() from the same parameters, Adam
   state and rollout: epochs run, Adam steps, parameters and losses, and the losses against eager runs of exactly the
   epochs that ran.  The eager hand-written update against autograd with the same stop."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl

pytestmark = pytest.mark.gpu
P = _native.ptr
LOSSES = ('policy_loss', 'value_loss', 'entropy', 'old_approx_kl', 'approx_kl', 'clipfrac')


def kl_stop(target, state, epoch=0, kl32=None, kl_sum=None, rows=0, handle=None):
    _native.check(_native.lib().pb_kl_stop(P(kl32), kl_sum, rows, P(target), epoch, P(state), handle or 0,
                                           int(handle is not None), _native.stream_ptr()))


def f32_neighbours(t):
    f = np.float32(t)
    return [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]


# ---- 1. the predicate ----------------------------------------------------------------------------------------------------
def test_kl_stop_decides_like_torch_from_an_fp32_scalar():
    dev = torch.device('cuda')
    cases = []
    for t in (0.1, 0.02, 0.0, 1e-30):
        for a in f32_neighbours(t) + [np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf)]:
            cases.append((float(a), t))
    kl = torch.tensor([a for a, _ in cases], dtype=torch.float32, device=dev)
    tgt = torch.tensor([t for _, t in cases], dtype=torch.float32, device=dev)
    states = torch.full((len(cases), 2), 7, dtype=torch.int32, device=dev)
    for i in range(len(cases)):
        kl_stop(tgt[i], states[i], kl32=kl[i])
    got = states.cpu().numpy()
    for i, (a, t) in enumerate(cases):
        want = bool(torch.tensor(a, dtype=torch.float32) > t)
        assert bool(got[i, 0]) == want, (a, t, got[i])
        assert got[i, 1] == (1 if want else 2), (a, t, got[i])


def test_kl_stop_forms_the_fused_loss_value_from_an_fp64_row():
    """kl_sum / rows rounded once to fp32 is (stats / m).float() of fused_ppo_loss: with the target at that value and one ulp
    either side the decisions are (stop, no stop, no stop), which pins the device's value to it bit for bit."""
    dev = torch.device('cuda')
    gen = torch.Generator(device='cpu').manual_seed(3)
    rows_list = [1, 3, 3000, 524288, 7]
    sums = [float(x) for x in torch.rand(len(rows_list), generator=gen, dtype=torch.float64) * 40]
    stats = torch.zeros(len(rows_list), 8, dtype=torch.float64, device=dev)
    stats[:, 4] = torch.tensor(sums, dtype=torch.float64)
    state = torch.zeros(3 * len(rows_list), 2, dtype=torch.int32, device=dev)
    targets, k = [], 0
    for r, (m, s) in enumerate(zip(rows_list, sums)):
        v = float((torch.tensor([s], dtype=torch.float64) / m).float())
        for t in f32_neighbours(v):
            targets.append((r, m, float(t), bool(torch.tensor(v, dtype=torch.float32) > float(t))))
    tgt = torch.tensor([t for _, _, t, _ in targets], dtype=torch.float32, device=dev)
    for k, (r, m, t, _) in enumerate(targets):
        kl_stop(tgt[k], state[k], kl_sum=C.c_void_p(stats.data_ptr() + 64 * r + 32), rows=m)
    got = state[:, 0].cpu().numpy()
    assert [bool(g) for g in got] == [w for _, _, _, w in targets]
    assert [w for _, _, _, w in targets][:3] == [True, False, False]

    # the statistics pb_ppo_loss writes for real rows vs fused_ppo_loss's approx_kl on the same rows
    torch.manual_seed(5)
    m, n_act = 1000, 4
    logits = torch.randn(m, n_act, device=dev)
    value = torch.randn(m, device=dev)
    act = torch.randint(0, n_act, (m,), device=dev)
    olp = torch.log_softmax(logits + 0.3 * torch.randn(m, n_act, device=dev), 1).gather(1, act[:, None])[:, 0]
    adv, ret, oval = torch.randn(m, device=dev), torch.randn(m, device=dev), torch.randn(m, device=dev)
    cfg = clean_pufferl.pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    _, st = clean_pufferl.fused_ppo_loss(logits, value, act, olp, adv, ret, oval, cfg)
    row = torch.zeros(8, dtype=torch.float64, device=dev)
    gl, gv = torch.empty(m, n_act, device=dev), torch.empty(m, device=dev)
    _native.check(_native.lib().pb_ppo_loss(
        P(logits), n_act, P(value), 1, P(act), P(olp), P(adv), P(ret), P(oval), m, n_act, C.c_float(0.1), 1,
        C.c_float(0.1), C.c_float(0.5), C.c_float(0.01), P(gl), n_act, P(gv), 1, P(row), _native.stream_ptr()))
    v = float(st[4])
    tgt = torch.tensor([float(t) for t in f32_neighbours(v)], device=dev)
    state = torch.zeros(3, 2, dtype=torch.int32, device=dev)
    for i in range(3):
        kl_stop(tgt[i], state[i], kl_sum=C.c_void_p(row.data_ptr() + 32), rows=m)
    assert state[:, 0].tolist() == [1, 0, 0], (v, row[4].item())


def test_kl_stop_state_stays_set_and_epoch_zero_starts_a_call():
    """Without a handle only state is written: epoch 0 (re)starts the call, a later decision after a stop changes nothing,
    epochs run counts the next epoch when it does not stop."""
    dev = torch.device('cuda')
    state = torch.tensor([5, 5], dtype=torch.int32, device=dev)
    big, small = torch.tensor(1.0, device=dev), torch.tensor(0.0, device=dev)
    tgt = torch.tensor([0.5], device=dev)
    kl_stop(tgt, state, epoch=0, kl32=small)
    assert state.tolist() == [0, 2]
    kl_stop(tgt, state, epoch=1, kl32=small)
    assert state.tolist() == [0, 3]
    kl_stop(tgt, state, epoch=2, kl32=big)
    assert state.tolist() == [1, 3]
    kl_stop(tgt, state, epoch=3, kl32=small)           # stays stopped
    assert state.tolist() == [1, 3]
    kl_stop(tgt, state, epoch=0, kl32=big)             # a new call
    assert state.tolist() == [1, 1]
    kl_stop(tgt, state, epoch=0, kl32=small)
    assert state.tolist() == [0, 2]


# ---- 2. the IF-node helpers ----------------------------------------------------------------------------------------------
def bump(step, zero):
    """A device counter advanced by a project kernel: pb_clip_adam's step += 1 on one parameter with a zero gradient and
    zero learning rate."""
    t = (_native.AdamTensor * 1)()
    t[0] = _native.AdamTensor(zero[0:].data_ptr(), zero[1:].data_ptr(), zero[2:].data_ptr(), step.data_ptr(),
                              zero[3:].data_ptr(), 1)
    _native.check(_native.lib().pb_clip_adam(t, 1, C.c_float(0.5), C.c_float(1.0), C.c_float(0.0), None, C.c_float(0.9),
                                             C.c_float(0.999), C.c_float(1e-5), None, _native.stream_ptr()))


def test_if_nodes_run_the_bodies_the_predicate_lets_run(monkeypatch):
    """IF{probe; decide(0)} -> IF{count; decide(1)} -> IF{count; decide(2)} -> IF{count}, each IF node on its own handle,
    as train() captures its epochs, replayed with the stop after epoch 0, 1, 2 or never, in an order where a replay that
    runs fewer bodies follows one that ran more: a handle left at 1 by the previous launch would run its body, so this
    checks that every launch starts with the later handles at 0 (and epoch 0's at 1).  Every handle is created from the
    capture stream, i.e. on the root graph that holds the IF nodes, none from the body stream.  Each body also allocates
    from the graph's pool (a torch op)."""
    dev = torch.device('cuda')
    lib = _native.lib()
    created = []
    create = lib.pb_graph_cond_create

    def spy(stream, default, out):
        created.append((stream.value, default))
        return create(stream, default, out)
    monkeypatch.setattr(lib, 'pb_graph_cond_create', spy)
    ks = clean_pufferl._KLStop(dev)
    kl = torch.zeros(3, device=dev)
    probe, count = torch.zeros((), device=dev), torch.zeros((), device=dev)
    zero = torch.zeros(4, device=dev)
    alloc_sum = torch.zeros(1, device=dev)
    ks.target.fill_(0.5)
    bump(count, zero)          # warm up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    ks.pool = torch.cuda.graph_pool_handle()
    with torch.cuda.graph(graph, pool=ks.pool):
        capture_stream = torch.cuda.current_stream().cuda_stream
        ks.begin(4)
        for e in range(4):
            with ks.if_body(e):
                bump(probe if e == 0 else count, zero)
                if e > 0:
                    alloc_sum.add_(torch.ones(1000, device=dev).sum())
                if e < 3:
                    ks.decide(e, approx_kl=kl[e])
    monkeypatch.undo()
    assert created == [(capture_stream, 1), (capture_stream, 0), (capture_stream, 0), (capture_stream, 0)], created
    assert capture_stream != ks.body.cuda_stream and len(set(ks.handles)) == 4, ks.handles
    for it, stop_after in enumerate((None, 0, 2, 1, None, 0)):
        kl.fill_(0.0)
        if stop_after is not None:
            kl[stop_after] = 1.0
        probe.zero_()
        count.zero_()
        alloc_sum.zero_()
        graph.replay()
        torch.cuda.synchronize()
        bodies = 3 if stop_after is None else stop_after
        assert float(probe) == 1.0, it
        assert float(count) == bodies and float(alloc_sum) == 1000.0 * bodies, (it, float(count), float(alloc_sum))
        assert ks.state.tolist() == [int(stop_after is not None), 1 + bodies], (it, ks.state.tolist())
    ks.close()


def test_helpers_refuse_to_run_outside_a_capture():
    lib = _native.lib()
    s = torch.cuda.Stream()
    body = torch.cuda.Stream()
    state, tgt, kl = torch.zeros(2, dtype=torch.int32, device='cuda'), torch.zeros(1, device='cuda'), torch.zeros(1, device='cuda')
    torch.cuda.synchronize()
    n0 = lib.pb_launch_count()
    h = C.c_uint64()
    sp, bp = C.c_void_p(s.cuda_stream), C.c_void_p(body.cuda_stream)
    assert lib.pb_graph_cond_create(sp, 0, C.byref(h)) == _native.PB_ERR_STATE
    assert lib.pb_graph_if_begin(1, sp, bp) == _native.PB_ERR_STATE
    assert lib.pb_graph_if_end(bp) == _native.PB_ERR_STATE
    assert lib.pb_graph_if_begin(1, sp, sp) == _native.PB_ERR_INVALID
    assert lib.pb_graph_if_begin(1, sp, None) == _native.PB_ERR_INVALID
    assert lib.pb_graph_cond_create(None, 0, C.byref(h)) == _native.PB_ERR_INVALID
    assert lib.pb_graph_cond_create(sp, 0, None) == _native.PB_ERR_INVALID
    assert lib.pb_kl_stop(P(kl), C.c_void_p(8), 1, P(tgt), 0, P(state), 0, 0, None) == _native.PB_ERR_INVALID   # two sources
    assert lib.pb_kl_stop(None, None, 1, P(tgt), 0, P(state), 0, 0, None) == _native.PB_ERR_INVALID             # none
    assert lib.pb_kl_stop(None, C.c_void_p(8), 0, P(tgt), 0, P(state), 0, 0, None) == _native.PB_ERR_INVALID    # rows 0
    assert lib.pb_kl_stop(P(kl), None, 0, None, 0, P(state), 0, 0, None) == _native.PB_ERR_INVALID              # no target
    assert lib.pb_launch_count() == n0


# ---- 3. train() ----------------------------------------------------------------------------------------------------------
def make_config(n, h, **kw):
    cfg = dict(seed=1, torch_deterministic=True, env='squared', batch_size=n * h, bptt_horizon=8, minibatch_size=n * h // 2,
               cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
               update_epochs=3, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5,
               ent_coef=0.01, max_grad_norm=0.5, target_kl=1e9, anneal_lr=False, total_timesteps=10 ** 9)
    cfg.update(kw)
    return clean_pufferl.pufferlib_b200.namespace(**cfg)


# name -> (env, num_envs, horizon, recurrent, config overrides, (engine, form))
COMBOS = {
    'mlp_fused_direct': ('breakout', 64, 128, False, {}, ('mlp_fused', 'direct')),
    'mlp_chain_slabs': ('squared', 64, 32, False, dict(fused_update=False), ('mlp_chain', 'slabs')),
    'packed_autograd': ('breakout', 64, 32, False, dict(manual_update=False), ('packed', 'slabs')),
    'bptt_segments': ('memory', 64, 32, True, {}, ('bptt', 'segments')),
}


def make_data(env, n, h, recurrent, kw):
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    if recurrent:
        net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
        pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=3, fused_update=True).cuda()
    else:
        pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=7).cuda()
    return clean_pufferl.create(make_config(n, h, env=env, **kw), vec, pol), pol


def adam_state(opt):
    return [opt.state[p][k] for p in opt.param_groups[0]['params'] for k in ('exp_avg', 'exp_avg_sq', 'step')]


class Snapshot:
    def __init__(self, data, pol):
        self.data, self.pol = data, pol
        self.params = [p.detach().clone() for p in pol.parameters()]
        self.adam = [t.clone() for t in adam_state(data.optimizer)]

    def restore(self):
        with torch.no_grad():
            for p, s in zip(self.pol.parameters(), self.params):
                p.copy_(s)
            for t, s in zip(adam_state(self.data.optimizer), self.adam):
                t.copy_(s)
        clean_pufferl._invalidate_policy_cache(self.data)


def result(data, pol):
    return dict(params=[p.detach().clone() for p in pol.parameters()], adam=[t.clone() for t in adam_state(data.optimizer)],
                losses={k: float(getattr(data.losses, k)) for k in LOSSES}, epochs=data.train_epochs_run,
                step=float(adam_state(data.optimizer)[2]))


def compare(got, ref, what):
    perr = max(float((a - b).abs().max()) for a, b in zip(got['params'], ref['params']))
    assert perr <= 2e-6, (what, perr)
    for i, (a, b) in enumerate(zip(got['adam'], ref['adam'])):
        if i % 3 == 2:
            assert torch.equal(a, b), (what, 'step', a, b)
        else:
            tol = (1e-3 if i % 3 == 0 else 1e-4) * float(b.abs().max()) + 1e-12
            assert float((a - b).abs().max()) <= tol, (what, i, float((a - b).abs().max()), tol)
    for k, v in ref['losses'].items():
        assert np.isclose(got['losses'][k], v, rtol=1e-4, atol=1e-4), (what, k, got['losses'][k], v)


def kl_probe(monkeypatch):
    """Records the approx_kl each pb_kl_stop decision reads (eager calls only)."""
    seen = []
    orig = clean_pufferl._KLStop.decide

    def spy(self, epoch, approx_kl=None, stats=None, row=0, rows=0):
        if approx_kl is not None:
            seen.append(float(approx_kl.detach()))
        else:
            seen.append(float((stats[row, 4] / rows).float()))
        return orig(self, epoch, approx_kl=approx_kl, stats=stats, row=row, rows=rows)
    monkeypatch.setattr(clean_pufferl._KLStop, 'decide', spy)
    return seen


def stop_targets(kls):
    """target_kl values that stop after epoch 0, after epoch 1 and never, from one eager run's approx_kl per epoch."""
    kl0, kl1 = kls[0], kls[1]
    assert 0 < kl0 < kl1 and kl1 - kl0 > 1e-3 * kl1, kls
    return {0: 0.5 * kl0, 1: 0.5 * (kl0 + kl1), None: 1e9}


@pytest.mark.parametrize('name', list(COMBOS))
def test_captured_train_with_target_kl_matches_eager_train(name, monkeypatch):
    env, n, h, recurrent, kw, plan_want = COMBOS[name]
    data, pol = make_data(env, n, h, recurrent, dict(kw, cuda_graph=True))
    for _ in range(2):                    # eager (initialises Adam), then capture + first replay
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
    assert data.train_graph_state == 2, data.msg
    plan = clean_pufferl.update_plan(data)
    assert (plan.engine, plan.form, plan.capture) == plan_want + ('whole',), plan
    clean_pufferl.evaluate(data)
    snap = Snapshot(data, pol)
    nm = data.experience.num_minibatches

    seen = kl_probe(monkeypatch)
    data.config.cuda_graph_train = False
    clean_pufferl.train(data)
    monkeypatch.undo()
    assert data.train_epochs_run == 3 and len(seen) == 2, seen
    targets = stop_targets(seen)

    replays = {}
    for stop in (None, 0, 1):
        want_epochs = 3 if stop is None else stop + 1
        data.config.target_kl = targets[stop]
        snap.restore()
        data.config.cuda_graph_train = False
        clean_pufferl.train(data)
        ref = result(data, pol)
        snap.restore()
        data.config.cuda_graph_train = True
        r0, l0 = data.train_graph_replays, _native.lib().pb_launch_count()
        clean_pufferl.train(data)
        assert data.train_graph_replays == r0 + 1 and _native.lib().pb_launch_count() == l0
        assert data.train_graph_state == 2
        got = replays[stop] = result(data, pol)
        print(f'[target_kl] {name} stop after {stop}: epochs {got["epochs"]}, losses {got["losses"]} vs {ref["losses"]}',
              flush=True)
        assert got['epochs'] == ref['epochs'] == want_epochs, (stop, got['epochs'], ref['epochs'])
        assert got['step'] - float(snap.adam[2]) == want_epochs * nm == ref['step'] - float(snap.adam[2])
        compare(got, ref, (name, stop))

    # two replays in a row, different stop epochs: the second holds nothing of the first's later epochs
    for stop in (1, 0):
        snap.restore()
        data.config.target_kl = targets[stop]
        clean_pufferl.train(data)
        again = result(data, pol)
        assert again['epochs'] == stop + 1
        compare(again, replays[stop], (name, 'back-to-back', stop))

    # the losses are the sums over the minibatches that ran: eager runs of exactly those epochs without target_kl
    data.config.cuda_graph_train = False
    for stop in (0, 1):
        snap.restore()
        data.config.target_kl, data.config.update_epochs = None, stop + 1
        clean_pufferl.train(data)
        assert data.train_epochs_run == stop + 1
        compare(result(data, pol), replays[stop], (name, 'epochs only', stop))
    clean_pufferl.close(data)


def test_eager_manual_update_with_target_kl_matches_autograd(monkeypatch):
    """The hand-written chain with target_kl (manual_update=True, eager) vs autograd + clip_grad_norm_ + torch.optim.Adam
    (manual_update=False), same rollout: the same stop epoch, parameters within 2e-5, losses within 1e-4 relative."""
    n, h = 64, 32

    def run(manual, target):
        data, pol = make_data('breakout', n, h, False, dict(manual_update=manual, fused_update=False, cuda_graph=False,
                                                             target_kl=target))
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        out = dict(params=[p.detach().cpu().clone() for p in pol.parameters()],
                   losses=np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy,
                                    data.losses.approx_kl, data.losses.clipfrac, data.losses.explained_variance]),
                   epochs=data.train_epochs_run, used=data.manual_update is not None,
                   steps=[float(data.optimizer.state[p]['step']) for p in pol.parameters()])
        clean_pufferl.close(data)
        return out
    seen = kl_probe(monkeypatch)
    run(True, 1e9)
    monkeypatch.undo()
    t = stop_targets(seen)[1]
    a, b = run(True, t), run(False, t)
    assert a['used'] and not b['used']
    assert a['epochs'] == b['epochs'] == 2, (a['epochs'], b['epochs'])
    assert a['steps'] == b['steps'] == [4.0] * 6
    diff = max(float((x - y).abs().max()) for x, y in zip(a['params'], b['params']))
    assert diff <= 2e-5, diff
    assert np.allclose(a['losses'], b['losses'], rtol=1e-4, atol=1e-6), (a['losses'], b['losses'])
