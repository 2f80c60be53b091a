"""The persistent rollout kernel (k_breakout_rollout, pb_rollout_breakout_mlp) at its launch boundaries: horizons 1, 3 and
17 (the last tile and the carry store in the other buffer, barrier phases of odd H), one CTA and several, grids with more
CTAs than SMs (a second wave), the benchmark's 16 384 envs x 128 steps, resets inside and across launches, rollouts that
alternate with the per-step loop (k_breakout + pb_policy_mlp_sample), env shards (env_index_offset), and the launcher's
refusals.

Every rollout is checked in full: env rows and the closing step's outputs replayed bit for bit through the oracle with the
kernel's actions; values, logprobs and sampled actions on every row; the step-0 dump of the hidden layer and the heads.

The encoder weights are put on a grid of 2^-8 (|w| < 0.09).  The observations are multiples of 2^-8 below 1, so every
partial sum of obs . W_enc^T is a multiple of 2^-16 below 16: exact in fp32 whatever order the tensor core adds in.  The
kernel's relu(h) is then fl(sum + b_enc), one fp32 rounding, known bit for bit on every row; what is left to bound is the
fp32 accumulation of the head products (util_gpu.ACC_F32).  The rest of the policy is left at full precision: the biases
at their random init, the heads scaled so the policies are far from uniform."""
import ctypes as C

import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
from pufferlib_b200 import _native, clean_pufferl, models
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from oracle.envs import OracleVec
from util_gpu import check_rollout_dump, rollout_heads_ref, restated_draw, softmax64, uniforms

pytestmark = pytest.mark.gpu
N_ACT = 4
WINDOW = 1e-4        # rows whose uniform lies this close to an inner CDF boundary may draw either neighbour
# fp32 sampling epilogue (pb_sample_row: expf / logf within 2 ulp, a handful of fp32 adds): at most 2^-19 of the
# magnitudes involved
EPI = 2.0 ** -19


def cpu(x):
    return x.detach().cpu().numpy()


def sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def make(n, h, env_kwargs=None, backend=pvec.B200, seed=5):
    vec = pvec.make(ocean.env_creator('breakout'), env_kwargs=env_kwargs or {}, num_envs=n, backend=backend)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=seed).cuda()
    model = pol.policy
    with torch.no_grad():
        model.encoder.weight.copy_(torch.round(model.encoder.weight * 256) / 256)     # the grid of the module docstring
        model.decoder.weight.mul_(40.0)             # the default init gives almost uniform policies
        model.decoder.bias.uniform_(-0.5, 0.5)
        model.value_head.weight.mul_(3.0)
    assert float(model.encoder.weight.detach().abs().max()) < 0.09
    cfg = pufferlib_b200.namespace(
        seed=1, torch_deterministic=True, env='breakout', batch_size=n * h, bptt_horizon=1, minibatch_size=n * h,
        cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
        update_epochs=1, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01,
        max_grad_norm=0.5, target_kl=None, anneal_lr=False, total_timesteps=10 ** 9, cuda_graph=False, fused_rollout=True)
    return clean_pufferl.create(cfg, vec, pol), vec, pol


def replay(ora, data, n, h):
    """Replay the rollout's actions through the oracle: obs / reward / done rows bit for bit, then the closing step's
    outputs in the vecenv's own buffers (row 0 of the next rollout).  -> the oracle's infos of the H steps."""
    exp, buf = data.experience, data.vecenv.buf
    acts, obs = cpu(exp.actions).reshape(h, n), cpu(exp.obs).reshape(h, n, 128)
    rew, done = cpu(exp.rewards).reshape(h, n), cpu(exp.dones).reshape(h, n)
    eps = []
    for t in range(h):
        o, r, d, _, _, _, _ = ora.recv()
        assert np.array_equal(o, obs[t]), f'obs row {t}: envs {np.nonzero((o != obs[t]).any(1))[0][:8]}'
        assert np.array_equal(r.view(np.uint32), rew[t].view(np.uint32)), f'rewards row {t}'
        assert np.array_equal(d.astype(np.float32), done[t]), f'dones row {t}'
        ora.send(acts[t])
        eps += ora.infos
    o, r, d, _, _, _, _ = ora.recv()
    assert np.array_equal(o, cpu(buf.observations)), 'closing step: observations'
    assert np.array_equal(r.view(np.uint32), cpu(buf.rewards).view(np.uint32)), 'closing step: rewards'
    assert np.array_equal(d, cpu(buf.terminals)), 'closing step: terminals'
    assert np.array_equal(d.astype(np.float32), cpu(buf.dones_f32)), 'closing step: dones_f32'
    return eps


def check_stats(stats, eps):
    """evaluate()'s device-side EpisodeStats means against the oracle's infos for the same steps."""
    if not eps:
        assert 'episode_return' not in stats, stats
        return
    assert np.isclose(stats['episode_return'], np.mean([i['episode_return'] for i in eps]), rtol=1e-9, atol=0)
    assert np.isclose(stats['episode_length'], np.mean([i['episode_length'] for i in eps]), rtol=1e-9, atol=0)
    assert np.isclose(stats['score'], np.mean([i['score'] for i in eps]), rtol=1e-6, atol=0)


def check_policy(data, n, h, offset0, rep):
    """Values, logprobs and actions of every row of the rollout against fp64 math on its stored observations.  relu(h) is
    exact (module docstring), so the heads are within rollout_heads_ref's bound b of the fp64 outputs z: the value within
    b_value, the logprob z_a - lse within |dz_a| + max_k |dz_k| <= 2 max_k b_k plus the fp32 epilogue.  Actions: the
    inverse-CDF draw of the uniform of (seed, offset0 + t, e) on the fp64 probabilities, except rows within WINDOW of a
    boundary."""
    exp, pol = data.experience, data.policy
    model = pol.policy
    w_enc, b_enc = model.encoder.weight.detach().double(), model.encoder.bias.detach().double()
    acts = cpu(exp.actions).reshape(h, n)
    with torch.no_grad():
        w_cat, b_cat = model.head_matrix()
        for t in range(h):
            rows = slice(t * n, (t + 1) * n)
            hid = torch.relu(exp.obs[rows].double() @ w_enc.t() + b_enc).float()      # exact: fl(sum + b_enc)
            out, bound = rollout_heads_ref(hid, w_cat, b_cat)
            dv = (exp.values[rows].double() - out[:, N_ACT]).abs()
            assert bool((dv <= bound[:, N_ACT]).all()), f'values row {t}: max err {float(dv.max()):.3e}'
            logits = out[:, :N_ACT]
            lse = logits.logsumexp(-1)
            lp = logits.gather(-1, exp.actions[rows].view(-1, 1)).squeeze(-1) - lse
            tol = 2 * bound[:, :N_ACT].amax(-1) + EPI * (1 + logits.abs().amax(-1) + lp.abs())
            dl = (exp.logprobs[rows].double() - lp).abs()
            assert bool((dl <= tol).all()), f'logprobs row {t}: max err {float(dl.max()):.3e}'
            want, near = restated_draw(softmax64(logits), uniforms(pol._seed, offset0 + t, n), WINDOW)
            bad = int(((want != acts[t]) & ~near).sum())
            assert bad == 0, f'actions row {t}: {bad} off the restated draw'
            rep['err_value'] = max(rep.get('err_value', 0.0), float(dv.max()))
            rep['tol_value'] = max(rep.get('tol_value', 0.0), float(bound[:, N_ACT].max()))
            rep['err_logprob'] = max(rep.get('err_logprob', 0.0), float(dl.max()))
            rep['tol_logprob'] = max(rep.get('tol_logprob', 0.0), float(tol.max()))
            rep['near'] = rep.get('near', 0) + int(near.sum())
            rep['rows'] = rep.get('rows', 0) + n


def rearm(data):
    """What train() does to the rollout buffer before the next evaluate() (Experience.sort_training_data), without an
    update: the weights stay as they are."""
    data.experience.sort_training_data()


def run_rollouts(data, ora, n, h, k, fused=(True,), rep=None):
    """k rollouts through clean_pufferl.evaluate, rollout i on the persistent kernel when fused[i % len(fused)] (else on
    the per-step loop), each checked in full against the oracle `ora` (which stays in lockstep across them).  The first
    fused rollout runs with the step-0 dump on (the kernel's DBG instance), the others as the product path runs them."""
    rep = {} if rep is None else rep
    pol, model = data.policy, data.policy.policy
    dbg_h = torch.full((n, 128), float('nan'), device='cuda')
    dbg_o = torch.full((n, 8), float('nan'), device='cuda')
    steps, dumped = 0, False
    try:
        for i in range(k):
            use_fused = fused[i % len(fused)]
            data.config.fused_rollout = use_fused
            dump = use_fused and not dumped
            if dump:
                _native.check(_native.lib().pb_rollout_debug_buffers(_native.ptr(dbg_h), _native.ptr(dbg_o)))
            f0 = getattr(data, 'fused_rollouts', 0)
            stats, _ = clean_pufferl.evaluate(data)
            if dump:
                _native.check(_native.lib().pb_rollout_debug_buffers(None, None))
                dumped = True
            assert getattr(data, 'fused_rollouts', 0) == f0 + (1 if use_fused else 0), 'the persistent kernel must run'
            assert data.experience.ptr == n * h
            eps = replay(ora, data, n, h)
            check_stats(stats, eps)
            rep['episodes'] = rep.get('episodes', 0) + len(eps)
            rep.setdefault('segment_episodes', []).append(len(eps))
            if use_fused:
                if dump:
                    r = check_rollout_dump(dbg_h, dbg_o, data.experience.obs[:n], model, exact_encoder=True)
                    assert bool((data.experience.values[:n] == dbg_o[:, N_ACT]).all()), 'stored values != dumped heads'
                    rep['dump'] = r
                check_policy(data, n, h, steps, rep)
            steps += h
            assert int(cpu(pol._counter)[0]) == steps
            rearm(data)
    finally:
        _native.lib().pb_rollout_debug_buffers(None, None)
    print(f'[rollout n={n} H={h} x{k}] values max err {rep["err_value"]:.2e} (bound <= {rep["tol_value"]:.2e}), logprobs '
          f'{rep["err_logprob"]:.2e} (<= {rep["tol_logprob"]:.2e}); step-0 relu(h) {rep["dump"][0]:.1e} '
          f'(bound <= {rep["dump"][1]:.1e}, bit-exact), heads {rep["dump"][2]:.2e} (<= {rep["dump"][3]:.2e}); '
          f'{rep["near"]} of {rep["rows"]} rows near a CDF boundary; {rep["episodes"]} episodes', flush=True)
    return rep


@pytest.mark.parametrize('n', [128, 384])
@pytest.mark.parametrize('h', [1, 3, 17])
def test_rollout_horizons(n, h):
    """Odd and single-step horizons: the closing step's tile and the carry store sit in the other buffer and barrier phase
    than at even H; three rollouts, so each starts from the state, carry rows and counter the previous one left."""
    data, vec, pol = make(n, h)
    ora = OracleVec('breakout', n)
    ora.async_reset(1)
    run_rollouts(data, ora, n, h, 3)
    clean_pufferl.close(data)


def test_rollout_second_wave():
    """128 (SMs + 3) envs: the kernel runs one CTA per SM, so the last three CTAs start only when others have finished."""
    n, h = 128 * (sms() + 3), 17
    data, vec, pol = make(n, h)
    ora = OracleVec('breakout', n)
    ora.async_reset(1)
    run_rollouts(data, ora, n, h, 2)
    clean_pufferl.close(data)


def test_rollout_short_episodes_second_wave():
    """max_ticks = 25 with a second wave: episodes end every 26 steps, inside each launch and across its boundaries
    (H = 48), so the done flags, the auto-resets and the running episode return / length are carried through HBM."""
    n, h = 128 * (sms() + 3), 48
    data, vec, pol = make(n, h, env_kwargs={'max_ticks': 25})
    ora = OracleVec('breakout', n, iparam=[25])
    ora.async_reset(1)
    rep = run_rollouts(data, ora, n, h, 3)
    assert rep['episodes'] >= 4 * n
    clean_pufferl.close(data)


def test_rollout_benchmark_shape():
    """bench.py's rollout: 16 384 envs x 128 steps (128 CTAs), default max_ticks, two rollouts so episodes cross the
    rollout boundary."""
    n, h = 16384, 128
    data, vec, pol = make(n, h)
    ora = OracleVec('breakout', n)
    ora.async_reset(1)
    run_rollouts(data, ora, n, h, 2)
    clean_pufferl.close(data)


def test_rollout_alternates_with_per_step_loop():
    """fused, per-step, fused, per-step on the same data / vecenv: each path must take over exactly the state the other
    wrote back (env state, done flags, carry rows, running episode return / length, draw counter).  max_ticks = 10, so
    episodes end in every segment and cross every switch."""
    n, h = 384, 24
    data, vec, pol = make(n, h, env_kwargs={'max_ticks': 10})
    ora = OracleVec('breakout', n, iparam=[10])
    ora.async_reset(1)
    rep = run_rollouts(data, ora, n, h, 4, fused=(True, False))
    assert data.fused_rollouts == 2 and all(e > 0 for e in rep['segment_episodes']), rep['segment_episodes']
    clean_pufferl.close(data)


def test_rollout_env_shards():
    """env_index_offset (one shard of a multi-GPU run): envs seeded by global index on the persistent kernel, replayed
    through an oracle shard with the same offset; two offsets must give different rollouts."""
    n, h = 256, 32
    obs = {}
    for k in (1, 3):
        data, vec, pol = make(n, h, backend=pvec.B200.options(env_index_offset=k * n))
        ora = OracleVec('breakout', n, env_index_offset=k * n)
        ora.async_reset(1)
        run_rollouts(data, ora, n, h, 2)
        obs[k] = cpu(data.experience.obs)
        clean_pufferl.close(data)
    assert not np.array_equal(obs[1], obs[3])


def test_rollout_refusals():
    """pb_rollout_breakout_mlp refuses bad arguments before it launches anything: the return code, no kernel launched, and
    the rollout tensors, the vecenv's buffers and the draw counter untouched."""
    n, h = 256, 4
    lib = _native.lib()
    data, vec, pol = make(n, h)
    model = pol.policy
    fresh = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200)         # never reset
    ragged = pvec.make(ocean.env_creator('breakout'), num_envs=200, backend=pvec.B200)
    ragged.async_reset(1)
    torch.cuda.synchronize()
    dev = torch.device('cuda')
    rows = dict(obs=torch.full((h * n + 1, 128), -7.0, device=dev), rewards=torch.full((h * n,), -7.0, device=dev),
                dones=torch.full((h * n,), -7.0, device=dev), values=torch.full((h * n,), -7.0, device=dev),
                logprobs=torch.full((h * n,), -7.0, device=dev), actions=torch.full((h * n,), -7, dtype=torch.int64, device=dev))
    w_enc = torch.zeros(128 * 128 + 4, device=dev)
    w_enc[:128 * 128] = model.encoder.weight.detach().reshape(-1)
    with torch.no_grad():
        w_cat, b_cat = model.head_matrix()
    counter = torch.full((1,), 11, dtype=torch.int64, device=dev)
    before = {k: v.clone() for k, v in rows.items()}
    own = {k: v.clone() for k, v in vec.buf.items()}

    def call(v, horizon=h, obs_off=0, w_off=0, n_act=N_ACT, carry_edit=None):
        carry = v._env_out(None)
        if carry_edit:
            carry_edit(carry)
        return lib.pb_rollout_breakout_mlp(
            v._handle, horizon, C.c_void_p(rows['obs'].data_ptr() + obs_off), _native.ptr(rows['rewards']),
            _native.ptr(rows['dones']), _native.ptr(rows['values']), _native.ptr(rows['logprobs']),
            _native.ptr(rows['actions']), C.byref(carry), C.c_void_p(w_enc.data_ptr() + w_off),
            _native.ptr(model.encoder.bias), _native.ptr(w_cat), _native.ptr(b_cat), n_act, C.c_uint64(pol._seed),
            _native.ptr(counter), _native.stream_ptr())

    def no_dones(carry):
        carry.dones_f32 = None

    def wide_rows(carry):
        carry.obs_stride = 1024

    cases = [('no reset', lambda: call(fresh), _native.PB_ERR_STATE, 'reset() first'),
             ('num_envs % 128', lambda: call(ragged), _native.PB_ERR_UNSUPPORTED, 'multiple of 128'),
             ('horizon 0', lambda: call(vec, horizon=0), _native.PB_ERR_INVALID, 'bad horizon'),
             ('horizon -1', lambda: call(vec, horizon=-1), _native.PB_ERR_INVALID, 'bad horizon'),
             ('horizon * n > 2^31 - 1', lambda: call(vec, horizon=(1 << 31) // n), _native.PB_ERR_INVALID, 'bad horizon'),
             ('n_act 3', lambda: call(vec, n_act=3), _native.PB_ERR_INVALID, 'actions'),
             ('n_act 5', lambda: call(vec, n_act=5), _native.PB_ERR_INVALID, 'actions'),
             ('obs misaligned', lambda: call(vec, obs_off=4), _native.PB_ERR_INVALID, 'aligned'),
             ('W_enc misaligned', lambda: call(vec, w_off=4), _native.PB_ERR_INVALID, 'aligned'),
             ('carry obs_stride 1024', lambda: call(vec, carry_edit=wide_rows), _native.PB_ERR_INVALID, 'aligned'),
             ('no carry dones_f32', lambda: call(vec, carry_edit=no_dones), _native.PB_ERR_INVALID, 'dones_f32')]
    for name, fn, code, msg in cases:
        launches = lib.pb_launch_count()
        rc = fn()
        assert rc == code, (name, rc, _native.last_error())
        assert msg in _native.last_error(), (name, _native.last_error())
        assert lib.pb_launch_count() == launches, name
    torch.cuda.synchronize()
    for k, v in rows.items():
        assert torch.equal(v, before[k]), k
    for k, v in vec.buf.items():
        assert torch.equal(v, own[k]), k
    assert int(counter[0]) == 11
    # the same arguments, made valid, do launch: the refusals above were the arguments, not the set-up
    launches = lib.pb_launch_count()
    assert call(vec) == _native.PB_OK
    torch.cuda.synchronize()
    assert lib.pb_launch_count() == launches + 2 and int(counter[0]) == 11 + h
    assert not torch.equal(rows['actions'], before['actions'])
    fresh.close()
    ragged.close()
    clean_pufferl.close(data)
