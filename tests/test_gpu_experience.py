"""Experience (store -> GAE -> flatten_batch -> adv-norm) on the device vs the reference's own outputs
(tests/golden/experience_*.npz) and the numpy oracle; plus the standalone train-prep kernels at larger sizes."""
import numpy as np
import pytest
import torch

import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl
from pufferlib_b200.environments import ocean
from oracle import experience as oexp
from oracle import gae as ogae

pytestmark = pytest.mark.gpu


def cpu(x):
    return x.detach().cpu().numpy()


@pytest.mark.parametrize('case', ['experience_c1', 'experience_small', 'experience_one_mb'])
@pytest.mark.parametrize('bound', [True, False])
def test_experience_pipeline_vs_reference(golden, case, bound):
    g = golden(case)
    n, h = int(g['num_envs']), int(g['horizon'])
    vec = pvec.make(ocean.env_creator('squared'), num_envs=n, backend=pvec.B200)
    vec.async_reset(int(g['seed']))
    exp = clean_pufferl.Experience(n * h, int(g['bptt']), int(g['minibatch_size']), (7, 7), np.float32, ())
    if bound:
        vec.bind_rollout(exp)
    dev = torch.device('cuda')
    t = 0
    while not exp.full:
        o, r, d, tr, infos, env_id, mask = vec.recv()
        a = torch.as_tensor(g['tape'][t], device=dev)
        exp.store(o, torch.as_tensor(g['values_in'][t], device=dev), a, torch.as_tensor(g['logprobs_in'][t], device=dev),
                  r, d, env_id, mask)
        vec.send(a)
        t += 1
    assert t == h
    # stored rollout == the reference's Experience arrays, bit for bit
    assert np.array_equal(cpu(exp.obs), g['stored_obs_i8'].astype(np.float32))
    for k in ('actions', 'logprobs', 'rewards', 'dones', 'values'):
        assert np.array_equal(cpu(getattr(exp, k)), g['stored_' + k]), k
    idxs = exp.sort_training_data()
    assert np.array_equal(np.asarray(idxs), g['idxs'])
    adv = cpu(exp.compute_gae(float(g['gamma']), float(g['gae_lambda'])))
    ref = g['advantages']
    assert np.max(np.abs(adv - ref) / np.maximum(1.0, np.abs(ref))) <= 1e-5
    exp.flatten_batch()
    assert np.array_equal(cpu(exp.b_obs), g['b_obs_i8'].astype(np.float32))
    for k in ('b_actions', 'b_logprobs', 'b_dones', 'b_values'):
        assert np.array_equal(cpu(getattr(exp, k)), g[k]), k
    for k in ('b_advantages', 'b_returns'):
        assert np.allclose(cpu(getattr(exp, k)), g[k], rtol=1e-5, atol=1e-5), k
    assert np.allclose(cpu(exp.returns), g['returns_np'], rtol=1e-5, atol=1e-5)      # the literal :476 quantity
    norm = cpu(exp.normalize_advantages())
    assert np.allclose(norm, g['b_advantages_normalized'], rtol=1e-5, atol=2e-5)
    # a second rollout through the same buffers: carry-over row 0 must be the step that closed the first rollout
    o2 = vec.recv()[0]
    assert cpu(o2).shape == (n, 7, 7)
    vec.close()


@pytest.mark.parametrize('n,h,mb,bptt,obs_shape,dtype', [
    (64, 128, 2048, 16, (7, 7), np.float32), (33, 12, 36, 4, (5,), np.float32), (16, 64, 256, 8, (128,), np.float32),
    (8, 32, 64, 16, (4, 84, 84), np.uint8), (100, 10, 250, 5, (3,), np.uint8), (256, 128, 4096, 32, (116,), np.float32)])
def test_flatten_and_gather_vs_numpy_oracle(n, h, mb, bptt, obs_shape, dtype):
    rng = np.random.default_rng(n * h)
    b = n * h
    dev = torch.device('cuda')
    exp = clean_pufferl.Experience(b, bptt, mb, obs_shape, dtype, ())
    ora = oexp.Experience(b, bptt, mb, obs_shape, dtype)
    if np.dtype(dtype) == np.uint8:
        obs = rng.integers(0, 256, size=(b, *obs_shape), dtype=np.uint8)
    else:
        obs = rng.standard_normal((b, *obs_shape)).astype(np.float32)
    fields = dict(actions=rng.integers(0, 6, size=b).astype(np.int64), logprobs=-rng.random(b).astype(np.float32),
                  rewards=rng.standard_normal(b).astype(np.float32), dones=(rng.random(b) < 0.05).astype(np.float32),
                  values=rng.standard_normal(b).astype(np.float32))
    exp.obs.copy_(torch.as_tensor(obs, device=dev))
    ora.obs[:] = obs
    for k, v in fields.items():
        getattr(exp, k).copy_(torch.as_tensor(v, device=dev))
        getattr(ora, k)[:] = v
    exp.num_envs = n
    ora.sort_keys = [(e, t) for t in range(h) for e in range(n)]
    idxs = ora.sort_training_data()
    assert np.array_equal(np.asarray(exp.sort_training_data()), idxs)
    adv_ref = ogae.compute_gae(ora.dones[idxs], ora.values[idxs], ora.rewards[idxs], 0.99, 0.95)
    adv = cpu(exp.compute_gae(0.99, 0.95))
    assert np.max(np.abs(adv - adv_ref) / np.maximum(1.0, np.abs(adv_ref))) <= 1e-5
    # feed the oracle's advantages so the remaining comparisons are exact byte movement
    exp.advantages.copy_(torch.as_tensor(adv_ref, device=dev))
    exp.flatten_batch()
    ora.flatten_batch(adv_ref)
    assert np.array_equal(cpu(exp.b_obs), ora.b_obs)
    for k in ('b_actions', 'b_logprobs', 'b_dones', 'b_values', 'b_advantages', 'b_returns'):
        assert np.array_equal(cpu(getattr(exp, k)), getattr(ora, k)), k
    assert np.array_equal(cpu(exp.returns), ora.returns_np)
    norm = cpu(exp.normalize_advantages())
    for m in range(exp.num_minibatches):
        t_ref = torch.as_tensor(ora.b_advantages[m])
        t_ref = ((t_ref - t_ref.mean()) / (t_ref.std() + 1e-8)).numpy()      # clean_pufferl.py:213 on CPU fp32
        assert np.allclose(norm[m], t_ref, rtol=1e-5, atol=2e-5)
    # zero-copy minibatch form: same row sets as the reference minibatches, slab-major order inside a minibatch
    nm, s_per_env = exp.num_minibatches, h // bptt
    ok = exp.flatten_batch_slabs()
    assert ok == (h % bptt == 0 and s_per_env % nm == 0)
    if ok:
        g_ = s_per_env // nm
        sl = exp._slabs
        for name in ('actions', 'logprobs', 'values', 'advantages', 'returns'):
            s_x, b_x = cpu(getattr(sl, name)), cpu(getattr(exp, 'b_' + name))
            for m in range(nm):
                assert np.array_equal(s_x[m].reshape(g_, bptt, n).transpose(2, 0, 1), b_x[m].reshape(n, g_, bptt)), name
        for m in range(nm):
            so = exp.slab_obs(m)
            assert so.data_ptr() == exp.obs.data_ptr() + m * bptt * n * exp.obs_row_bytes     # a view, not a copy
            assert np.array_equal(cpu(so).reshape(g_, bptt, n, -1).transpose(2, 0, 1, 3),
                                  cpu(exp.b_obs[m]).reshape(n, g_, bptt, -1))
        assert np.array_equal(cpu(exp.returns), ora.returns_np)
        norm_s = cpu(exp.normalize_advantages(slabs=True))
        for m in range(nm):
            assert np.allclose(norm_s[m].reshape(g_, bptt, n).transpose(2, 0, 1).reshape(-1), norm[m].reshape(-1),
                               rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize('n_mb,mb_size', [(1, 2), (1, 2048), (4, 65536), (2, 1048576), (3, 1000), (128, 16384)])
def test_adv_norm_vs_torch(n_mb, mb_size):
    dev = torch.device('cuda')
    g = torch.Generator(device='cpu').manual_seed(n_mb * 7 + mb_size)
    a = (torch.randn(n_mb, mb_size, generator=g) * 3 + 0.5).to(dev)
    out = torch.empty_like(a)
    lib = _native.lib()
    ws = torch.zeros(max(16, lib.pb_adv_norm_workspace_bytes(n_mb, mb_size)), dtype=torch.uint8, device=dev)
    _native.check(lib.pb_adv_norm(_native.ptr(a), _native.ptr(out), n_mb, mb_size, _native.ptr(ws), ws.numel(),
                                  _native.stream_ptr()))
    ref = torch.stack([(x - x.mean()) / (x.std() + 1e-8) for x in a.double()]).float()
    assert torch.allclose(out, ref, rtol=1e-5, atol=1e-5)
    # idempotence-style property at any size: the output has mean 0 and unbiased std 1
    assert torch.allclose(out.double().mean(1), torch.zeros(n_mb, device=dev, dtype=torch.float64), atol=1e-5)
    if mb_size > 2:
        assert torch.allclose(out.double().std(1), torch.ones(n_mb, device=dev, dtype=torch.float64), atol=1e-4)
    # in-place
    _native.check(lib.pb_adv_norm(_native.ptr(a), _native.ptr(a), n_mb, mb_size, _native.ptr(ws), ws.numel(),
                                  _native.stream_ptr()))
    assert torch.equal(a, out)


def test_copy_rows_and_store():
    dev = torch.device('cuda')
    lib = _native.lib()
    for row_bytes, n_rows in [(196, 64), (512, 1000), (7, 33), (28224, 16), (16, 1)]:
        src = torch.randint(0, 256, (n_rows, row_bytes + 16), dtype=torch.uint8, device=dev)
        dst = torch.zeros(n_rows, row_bytes + 32, dtype=torch.uint8, device=dev)
        _native.check(lib.pb_copy_rows(_native.ptr(src), row_bytes + 16, _native.ptr(dst), row_bytes + 32, row_bytes,
                                       n_rows, _native.stream_ptr()))
        assert torch.equal(dst[:, :row_bytes], src[:, :row_bytes]) and int(dst[:, row_bytes:].sum()) == 0
    n = 1000
    v, lp = torch.randn(n, device=dev), torch.randn(n, device=dev)
    a = torch.randint(0, 8, (n,), device=dev)
    vr, lr, ar = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, dtype=torch.int64, device=dev)
    _native.check(lib.pb_rollout_store(_native.ptr(v), _native.ptr(lp), _native.ptr(a), _native.ptr(vr), _native.ptr(lr),
                                       _native.ptr(ar), n, _native.stream_ptr()))
    assert torch.equal(v, vr) and torch.equal(lp, lr) and torch.equal(a, ar)


def make_config(n, h, **kw):
    import pufferlib_b200
    cfg = dict(seed=1, torch_deterministic=True, env='squared', batch_size=n * h, bptt_horizon=8, minibatch_size=n * h // 2,
               cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
               update_epochs=2, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5,
               ent_coef=0.01, max_grad_norm=0.5, target_kl=None, anneal_lr=False, total_timesteps=10 ** 9)
    cfg.update(kw)
    return pufferlib_b200.namespace(**cfg)


def test_evaluate_train_loop_eager_graph_and_host_modes():
    """create / evaluate / train with the reference signatures: eager device rollout, CUDA-graph rollout and the
    host-buffer (numpy in/out) mode all produce finite losses, and the rollout they store replays bit-exactly
    through the oracle (same actions -> same obs / rewards / dones)."""
    from pufferlib_b200 import models
    from pufferlib_b200.frameworks import cleanrl
    from oracle.squared import SquaredSerial
    n, h = 64, 32
    for mode in ('eager', 'graph', 'host', 'host_graph'):
        # (per-step info dicts need the host after every env step: the captured host loop runs with the device-side statistics)
        backend = pvec.B200.options(host_buffers=mode.startswith('host'), exact_infos=(False if mode == 'host_graph' else None))
        vec = pvec.make(ocean.env_creator('squared'), num_envs=n, backend=backend)
        torch.manual_seed(0)
        pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=(mode != 'host'), seed=1).cuda()
        data = clean_pufferl.create(make_config(n, h, cuda_graph=mode.endswith('graph')), vec, pol)
        ora = SquaredSerial(n)
        ora.async_reset(1)
        for it in range(3):                      # iteration 2 is the first graph replay
            stats, infos = clean_pufferl.evaluate(data)
            exp = data.experience
            acts = cpu(exp.actions).reshape(h, n)
            obs, rew, don = cpu(exp.obs).reshape(h, n, 7, 7), cpu(exp.rewards).reshape(h, n), cpu(exp.dones).reshape(h, n)
            for t in range(h):
                o, r, d, _, _, _, _ = ora.recv()
                assert np.array_equal(o, obs[t]) and np.array_equal(r, rew[t]) and np.array_equal(d, don[t] > 0), (mode, it, t)
                ora.send(acts[t])
            clean_pufferl.train(data)
            assert np.isfinite(data.losses.policy_loss) and np.isfinite(data.losses.value_loss)
            assert data.global_step == (it + 1) * n * h
            assert 'episode_return' in stats
            if mode.startswith('host'):
                # the pinned host arrays hold the step that closed the rollout, the action array the last actions sent
                # (host_graph: every env step of the captured loop copies through them, no host code in between)
                hobs = vec.host_sync()[0]
                assert hobs.shape == (n, 7, 7) and np.isfinite(hobs).all()
                assert np.array_equal(vec._host_np.actions, acts[-1])
                assert vec.d2h_bytes >= (it + 1) * h * n * 49 and vec.h2d_bytes == (it + 1) * h * n * 8
        if mode.endswith('graph'):
            assert data.graph_replays == 2 and data.graph_launches > 0
        clean_pufferl.close(data)


def test_lstm_policy_path():
    """Recurrent policies (LSTMWrapper + RecurrentPolicy): state carried across env steps in evaluate and across
    bptt segments in train (clean_pufferl.py:100-105, 188-191)."""
    from pufferlib_b200 import models
    from pufferlib_b200.frameworks import cleanrl
    n, h = 32, 16
    vec = pvec.make(ocean.env_creator('squared'), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
    pol = cleanrl.RecurrentPolicy(net).cuda()
    data = clean_pufferl.create(make_config(n, h), vec, pol)
    assert data.experience.lstm_h.shape == (1, n, 128)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        assert float(data.experience.lstm_h.abs().sum()) > 0
        clean_pufferl.train(data)
        assert np.isfinite(data.losses.policy_loss) and np.isfinite(data.losses.entropy)
    clean_pufferl.close(data)


def test_graphed_training_matches_eager_training():
    """CUDA-graph rollout + CUDA-graph train update are the same computation as the eager loop.  Same config in both runs
    (so the same capturable Adam), graphs on vs off.  The comparison is made where chaos has not set in yet: the GAE
    look-back composes tile aggregates in a timing-dependent order (1e-7 differences run to run), and action sampling
    amplifies any parameter difference over iterations, so: the first graph-replayed rollout (iteration 2) samples the
    same actions as the eager one, and after the first graphed update the parameters agree to 2e-5."""
    from pufferlib_b200 import models
    from pufferlib_b200.frameworks import cleanrl
    n, h = 64, 32
    params, rollouts = {}, {}
    for mode in ('eager', 'graph'):
        vec = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200)
        torch.manual_seed(0)
        pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=7).cuda()
        g = mode == 'graph'
        data = clean_pufferl.create(make_config(n, h, env='breakout', cuda_graph=True, cuda_graph_rollout=g,
                                                cuda_graph_train=g, anneal_lr=True, total_timesteps=20 * n * h), vec, pol)
        rollouts[mode], params[mode] = [], []
        for it in range(3):
            clean_pufferl.evaluate(data)
            rollouts[mode].append(cpu(data.experience.actions).copy())
            clean_pufferl.train(data)
            params[mode].append([p.detach().cpu().clone() for p in pol.parameters()])
        if g:
            assert data.train_graph_state == 2 and data.train_graph_replays == 2 and data.graph_replays == 2, data.msg
        else:
            assert data.train_graph_state != 2 and data.graph_replays == 0
        clean_pufferl.close(data)
    agree = [float((a == b).mean()) for a, b in zip(rollouts['eager'], rollouts['graph'])]
    diffs = [max(float((a - b).abs().max()) for a, b in zip(pa, pb)) for pa, pb in zip(params['eager'], params['graph'])]
    assert agree[0] == 1.0 and agree[1] > 0.9995 and agree[2] > 0.98, (agree, diffs)
    assert diffs[0] <= 2e-6 and diffs[1] <= 2e-5, (agree, diffs)


def test_zero_copy_minibatches_match_gathered_minibatches():
    """train() on zero-copy slab minibatches (Experience.flatten_batch_slabs; observations never gathered) is the same
    update as train() on the gathered, sorted minibatches of the reference layout: same rollout, parameters after the
    first update agree to 2e-5 (row order inside a minibatch only changes the summation order)."""
    from pufferlib_b200 import models
    from pufferlib_b200.frameworks import cleanrl
    n, h = 64, 32
    params, acts, used = {}, {}, {}
    for zc in (True, False):
        vec = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200)
        torch.manual_seed(0)
        pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=7).cuda()
        data = clean_pufferl.create(make_config(n, h, env='breakout', zero_copy_minibatches=zc), vec, pol)
        clean_pufferl.evaluate(data)
        acts[zc] = cpu(data.experience.actions).copy()
        clean_pufferl.train(data)
        params[zc] = [p.detach().cpu().clone() for p in pol.parameters()]
        used[zc] = data.experience._slabs is not None
        assert np.isfinite(data.losses.policy_loss) and np.isfinite(data.losses.explained_variance)
        clean_pufferl.close(data)
    assert used[True] and not used[False]
    assert np.array_equal(acts[True], acts[False])
    diff = max(float((a - b).abs().max()) for a, b in zip(params[True], params[False]))
    assert diff <= 2e-5, diff


def test_lstm_parity_vs_reference(golden):
    """The recurrent path against the REFERENCE's own run (tests/golden/lstm_squared.npz: unmodified
    clean_pufferl.create/evaluate/train + models.LSTMWrapper + cleanrl.RecurrentPolicy on CPU, generate.py::gen_lstm).
    Same initial weights, same seed, the reference's sampled actions replayed: evaluate must store the same
    observations / values / logprobs and leave the same LSTM state (lstm_h[:, env_id] carry, clean_pufferl.py:100-105);
    train must give the same losses and parameters (bptt segments [rows, bptt, *obs], state carried across the
    minibatches of an epoch and reset per epoch, :176-191; models.py:64-111)."""
    import pufferlib_b200
    from pufferlib_b200 import models
    from pufferlib_b200.frameworks import cleanrl
    g = golden('lstm_squared')
    n, h, bptt, mbs, hid = (int(g[k]) for k in ('num_envs', 'horizon', 'bptt', 'minibatch_size', 'hidden'))
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False     # the golden is CPU fp32
    try:
        vec = pvec.make(ocean.env_creator('squared'), num_envs=n, backend=pvec.B200)
        net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env, hidden_size=hid), input_size=hid,
                                 hidden_size=hid)
        net.policy.fast_path = False

        class TapePolicy(cleanrl.RecurrentPolicy):
            """RecurrentPolicy that replays the reference's sampled actions in evaluate (sampling itself is
            torch.multinomial on the CPU generator there; the given-action branch of sample_logits is the same code)."""
            tape, t = torch.as_tensor(g['actions'].reshape(h, n), device='cuda'), 0

            def forward(self, x, state=None, action=None):
                if action is None:
                    action = self.tape[self.t]
                    self.t += 1
                return super().forward(x, state, action)

        pol = TapePolicy(net).cuda()
        sd = {k[len('init/'):]: torch.as_tensor(g[k]) for k in g.files if k.startswith('init/')}
        assert set(sd) == set(pol.state_dict()), 'module / parameter names follow the reference'
        pol.load_state_dict(sd)
        cfg = pufferlib_b200.namespace(
            seed=int(g['seed']), torch_deterministic=True, env='squared', batch_size=n * h, bptt_horizon=bptt,
            minibatch_size=mbs, cpu_offload=False, device='cuda', compile=False, learning_rate=float(g['learning_rate']),
            gamma=0.99, gae_lambda=0.95, update_epochs=int(g['update_epochs']), norm_adv=True, clip_coef=0.1,
            clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01, max_grad_norm=0.5, target_kl=None,
            anneal_lr=False, total_timesteps=10 ** 9)
        data = clean_pufferl.create(cfg, vec, pol)
        clean_pufferl.evaluate(data)
        exp = data.experience
        assert np.array_equal(cpu(exp.obs), g['obs_i8'].astype(np.float32))
        assert np.array_equal(cpu(exp.actions), g['actions'])
        assert np.array_equal(cpu(exp.rewards), g['rewards']) and np.array_equal(cpu(exp.dones), g['dones'])
        assert np.allclose(cpu(exp.values), g['values'], rtol=1e-4, atol=2e-6)
        assert np.allclose(cpu(exp.logprobs), g['logprobs'], rtol=1e-4, atol=2e-6)
        assert np.allclose(cpu(exp.lstm_h), g['lstm_h'], rtol=1e-4, atol=2e-6)
        assert np.allclose(cpu(exp.lstm_c), g['lstm_c'], rtol=1e-4, atol=2e-6)
        clean_pufferl.train(data)
        assert np.array_equal(cpu(exp.b_obs), g['b_obs_i8'].astype(np.float32))
        assert np.allclose(cpu(exp.b_advantages), g['advantages'], rtol=1e-4, atol=1e-5)
        for k in ('policy_loss', 'value_loss', 'entropy', 'old_approx_kl', 'approx_kl', 'clipfrac'):
            assert np.isclose(getattr(data.losses, k), float(g['loss_' + k]), rtol=2e-3, atol=2e-5), \
                (k, getattr(data.losses, k), float(g['loss_' + k]))
        assert np.isclose(data.losses.explained_variance, float(g['loss_explained_variance']), rtol=1e-3, atol=1e-4)
        # parameters after update_epochs x num_minibatches Adam steps (lr 2.5e-3): Adam normalises the gradient, so fp32
        # noise on near-zero gradients moves single elements by a fraction of lr -- the bulk must agree tightly
        diffs = []
        for k, v in pol.state_dict().items():
            d = np.abs(cpu(v) - g['after/' + k])
            assert d.max() < 1e-3, (k, d.max())
            diffs.append(d.ravel())
        diffs = np.concatenate(diffs)
        assert np.mean(diffs) < 2e-5 and np.quantile(diffs, 0.99) < 2e-4
        moved = np.concatenate([np.abs(g['after/' + k] - g['init/' + k]).ravel() for k in sd])
        assert np.mean(moved) > 50 * np.mean(diffs), 'the update itself is much larger than the disagreement'
        clean_pufferl.close(data)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32


@pytest.mark.parametrize('n,bptt,nm,kw', [
    (36, 8, 2, dict(update_epochs=2, anneal_lr=True, total_timesteps=4 * 36 * 128, max_grad_norm=1e-3)),
    (64, 16, 4, dict(update_epochs=2, norm_adv=False, max_grad_norm=1e9))], ids=['R288_clipped', 'R1024_raw_adv'])
def test_direct_slab_update_replays_through_gathered_minibatches(n, bptt, nm, kw):
    """train() on the benchmark's path -- the fused update reading the arrival-order rollout tensors in place
    (Experience.minibatch 'direct': row_slab_stride = nm * R, returns and advantage normalisation formed in the kernel), then
    pb_clip_adam_parts with the head rebuild in its last CTA -- replayed step by step from a snapshot of the rollout, the
    parameters and the Adam state: minibatch membership and advantages from the oracles in float64, the normalisation of
    clean_pufferl.py:211-213, pb_mlp_update_fused on contiguous gathered rows with explicit returns, pb_clip_adam (the
    single-CTA norm pass) and pb_pack_heads.  The same kernel runs on both sides, so only the order of fp32 sums and the
    fp32 vs fp64 advantages differ.  A: R = 288 (ragged tiles, 8 slabs), two epochs, annealed lr, every step clipped;
    B: R = 1024, raw advantages, no clipping.  With breakout's 4 actions, one 128-byte line of the value-head weight is
    updated by two CTAs of pb_clip_adam_parts (asserted below): a head matrix rebuilt from a stale copy of that line would
    change the next minibatch."""
    from pufferlib_b200 import models
    from pufferlib_b200.frameworks import cleanrl
    h = 128
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=7).cuda()
    cfg = make_config(n, h, env='breakout', bptt_horizon=bptt, minibatch_size=n * h // nm, **kw)
    data = clean_pufferl.create(cfg, vec, pol)
    norms = replay_direct_update(data)
    if cfg.max_grad_norm < 1:
        assert min(norms) > cfg.max_grad_norm, norms          # every step clipped
    else:
        assert max(norms) < cfg.max_grad_norm, norms
    clean_pufferl.close(data)


def replay_direct_update(data, exp_avg_tol=1e-4):
    """The body of test_direct_slab_update_replays_through_gathered_minibatches for a breakout `data` (models.Default,
    config.update_epochs x num_minibatches steps): evaluate + train once, evaluate, snapshot, train() on the 'direct' path,
    then the replay and its checks (exp_avg_tol: the bound on the first Adam moments, relative to each one's maximum).
    Returns the gradient norms the replay's pb_clip_adam computed, one per step."""
    import ctypes as C
    import util_update as uu
    cfg, pol = data.config, data.policy
    clean_pufferl.evaluate(data)
    n = data.experience.num_envs
    h, nm, bptt = cfg.batch_size // n, cfg.batch_size // cfg.minibatch_size, cfg.bptt_horizon
    clean_pufferl.train(data)                  # the Adam state exists and the learning rate is annealed once
    assert data.train_minibatch_path == 'direct'
    clean_pufferl.evaluate(data)
    exp, model, opt = data.experience, pol.policy, data.optimizer
    params = [model.encoder.weight, model.encoder.bias, model.decoder.weight, model.decoder.bias, model.value_head.weight,
              model.value_head.bias]
    assert uu.split_lines(params[2:], first=128 * 128 + 128) > 0
    mine = [p.detach().clone() for p in params]
    st = [{k: opt.state[p][k].clone() for k in ('exp_avg', 'exp_avg_sq', 'step')} for p in params]
    group = opt.param_groups[0]
    lr, (b1, b2), eps = float(group['lr']), group['betas'], group['eps']
    roll = {k: cpu(getattr(exp, k)).copy() for k in ('obs', 'actions', 'logprobs', 'values', 'rewards', 'dones')}
    clean_pufferl.train(data)
    assert data.train_minibatch_path == 'direct' and data.manual_update.used_fused

    # the replay
    dev = torch.device('cuda')
    lib, s = _native.lib(), _native.stream_ptr()
    n_act = model.decoder.weight.shape[0]
    ora = oexp.Experience(n * h, bptt, n * h // nm, (128,), np.float32)
    for k, v in roll.items():
        getattr(ora, k)[:] = v
    ora.sort_keys = [(e, t) for t in range(h) for e in range(n)]
    idx = ora.sort_training_data()
    ora.flatten_batch(ogae.compute_gae_f64(ora.dones[idx], ora.values[idx], ora.rewards[idx], cfg.gamma, cfg.gae_lambda))
    w_cat, b_cat = torch.zeros(8, 128, device=dev), torch.zeros(8, device=dev)

    def pack_heads(ps, wc, bc):
        _native.check(lib.pb_pack_heads(_native.ptr(ps[2]), _native.ptr(ps[3]), _native.ptr(ps[4]), _native.ptr(ps[5]), n_act,
                                        128, _native.ptr(wc), _native.ptr(bc), None, None, 0, s))
    pack_heads(mine, w_cat, b_cat)
    ws = uu.workspace(dev)
    loss_cfg = (cfg.clip_coef, int(cfg.clip_vloss), cfg.vf_clip_coef, cfg.vf_coef, cfg.ent_coef)
    stats, norms = torch.zeros(6, dtype=torch.float64, device=dev), []
    norm_out = torch.zeros(1, device=dev)
    m = n * h // nm
    t = lambda a, dtype=torch.float32: torch.as_tensor(np.ascontiguousarray(a).reshape(-1), device=dev).to(dtype)
    for epoch in range(cfg.update_epochs):
        for mb in range(nm):
            a64 = ora.b_advantages[mb].astype(np.float64)
            if cfg.norm_adv:
                a64 = (a64 - a64.mean()) / (a64.std(ddof=1) + 1e-8)
            x = torch.as_tensor(ora.b_obs[mb].reshape(m, 128), device=dev)
            gflat, st8 = uu.fused(x, 128, m, m, 1, mine[0], mine[1], w_cat, b_cat, t(ora.b_actions[mb], torch.int64),
                                  t(ora.b_logprobs[mb]), t(a64), t(ora.b_returns[mb]), t(ora.b_values[mb]), n_act, False,
                                  cfg=loss_cfg, ws=ws)[:2]
            stats += st8[:6]
            grads = uu.grad_views(gflat, n_act)
            arr = (_native.AdamTensor * 6)()
            for k in range(6):
                arr[k] = _native.AdamTensor(mine[k].data_ptr(), st[k]['exp_avg'].data_ptr(), st[k]['exp_avg_sq'].data_ptr(),
                                            st[k]['step'].data_ptr(), grads[k].data_ptr(), mine[k].numel())
            _native.check(lib.pb_clip_adam(arr, 6, C.c_float(cfg.max_grad_norm), C.c_float(1.0), C.c_float(lr), None,
                                           C.c_float(b1), C.c_float(b2), C.c_float(eps), _native.ptr(norm_out), s))
            pack_heads(mine, w_cat, b_cat)
            norms.append(float(norm_out))
    torch.cuda.synchronize()
    n_steps = cfg.update_epochs * nm
    errs = {}
    for k, p in enumerate(params):
        errs[f'param{k}'] = float((p.detach() - mine[k]).abs().max())
        for name in ('exp_avg', 'exp_avg_sq'):
            errs[f'{name}{k}'] = uu.rel(opt.state[p][name], st[k][name])
        assert float(opt.state[p]['step']) == float(st[k]['step']) == float(n_steps * 2)
    print('replay errors', {k: f'{v:.2e}' for k, v in errs.items()}, 'norms', norms)
    for k in range(6):
        # one Adam step moves a parameter by at most ~lr; the two sides agree to 1e-3 of that per step
        assert errs[f'param{k}'] <= 1e-3 * lr * n_steps, errs
        assert errs[f'exp_avg{k}'] <= exp_avg_tol and errs[f'exp_avg_sq{k}'] <= 1e-4, errs
    # the head matrix train() leaves is the packed form of its own parameters, bit for bit, and the replay's up to the above
    mu = data.manual_update
    w_ref, b_ref = torch.full_like(w_cat, 9.0), torch.full_like(b_cat, 9.0)
    pack_heads([p.detach() for p in params], w_ref, b_ref)
    torch.cuda.synchronize()
    assert torch.equal(mu.w_cat, w_ref) and torch.equal(mu.b_cat, b_ref)
    assert float((mu.w_cat - w_cat).abs().max()) <= 1e-3 * lr * n_steps
    # the reported losses: per-minibatch means / n_mb summed over the epochs (clean_pufferl.py:249-254)
    tot = (stats / (m * nm)).cpu().numpy()
    tot[1] *= 0.5
    got = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy, data.losses.old_approx_kl,
                    data.losses.approx_kl, data.losses.clipfrac])
    # the policy loss is a mean of O(1) terms that nearly cancel (normalised advantages have mean 0): fp32 vs fp64 advantages
    # move it by ~1e-7 of a term
    assert abs(got[0] - tot[0]) <= 1e-6, (got, tot)
    assert np.allclose(got[1:], tot[1:], rtol=1e-4, atol=0), (got, tot)
    return norms
