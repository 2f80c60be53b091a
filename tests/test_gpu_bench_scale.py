"""The update kernels against fp64 at the sizes the benchmarks run them.

1. k_mlp_update (pb_mlp_update_fused) on bench.py's minibatch: breakout, 16 384 envs x 128 steps, 4 minibatches, so one
   minibatch is G = 2 slabs of R = 262 144 rows, slab stride and row_slab_stride 4R.  On 132 SMs every CTA runs about 62
   of the 8 192 64-row tiles and the two-stage x ring wraps about 31 times; the schedule tests stop at 8 tiles per CTA.
   Minibatch 0 and minibatch 3, whose last slab and per-row arrays end flush with their allocations, with the stage-by-
   stage, end-to-end and sum-of-squares checks of tests/util_update.py and its bounds; and bitwise reproducibility.
2. train() on the benchmark workload itself (bench.ppo_config), captured, replayed step by step through the oracle's
   minibatches and fp64 advantages (test_gpu_experience.replay_direct_update).
3. The BPTT kernels at bench_lstm.py's minibatch, 32 768 segments x 16 steps, at H = 128 and 256.  At H = 256 the saved
   rows are 8 KiB, so the row of segment 16 384 starts at byte 2^31 of a 4 GiB buffer.

Each case prints its largest errors and its peak device memory (torch.cuda.max_memory_allocated).  Observed on an H100
80GB HBM3 at a 700 W power limit (9 cases, 23 s; DESIGN.md §4): section 1 hidden 6.2e-7, dOut 8.4e-7, dPre 9.4e-8,
dW_enc 8.7e-6, dW_heads 1.35e-5, db_enc 1.3e-7, db_heads 6.5e-8 of their maxima, end to end <= 1.04e-3, peak 5.5 GiB;
section 2 parameters 1.4e-6 apart, peak 1.7 GiB, 11 s; section 3 peak 7.2 GiB (H = 128) and 14.0 GiB (H = 256)."""
import time

import pytest
import torch

import util_update as uu

pytestmark = pytest.mark.gpu

R_BENCH = 16384 * 128 // 4 // 2       # rows per slab of one bench minibatch (G = 2)


class Peak:
    """Prints the wall time and the peak device memory of one case."""

    def __enter__(self):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        self.t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        print(f'    peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB, '
              f'{time.perf_counter() - self.t0:.1f} s', flush=True)


# ---- 1. k_mlp_update at the benchmark minibatch --------------------------------------------------------------------------
# (slab_rows, n_slabs, slab_stride, n_act, seed, keyword arguments of util_update.case)
BENCH_DIRECT = dict(nm=4, returns=False, adv_norm=True)
UPDATE_CASES = {
    'bench_mb0': (R_BENCH, 2, 4 * R_BENCH, 4, 31, dict(BENCH_DIRECT, mb=0)),
    'bench_mb3_flush': (R_BENCH, 2, 4 * R_BENCH, 4, 32, dict(BENCH_DIRECT, mb=3, x_tail=0)),
    'bench_mb3_flush_7act_alt': (R_BENCH, 2, 4 * R_BENCH, 7, 33, dict(BENCH_DIRECT, mb=3, x_tail=0, cfg=uu.CFG_ALT)),
    'one_slab_524288': (2 * R_BENCH, 1, 2 * R_BENCH, 4, 34, {}),
    'ragged_slabs_mb3_flush': (R_BENCH + 37, 2, 4 * (R_BENCH + 37), 4, 35, dict(BENCH_DIRECT, mb=3, x_tail=0)),
}


@pytest.mark.parametrize('name', list(UPDATE_CASES))
def test_update_at_the_benchmark_minibatch(name):
    """util_update.case at the benchmark's minibatch, with its bounds: hidden 2e-5, dOut 2e-4, dPre 1e-5, the stage
    gradients 2e-5, end to end 5e-3, statistics 2e-3, the sums of squares 1e-12.

    What fp32 accumulation costs here: each CTA's dW_enc^T accumulator (wgmma, fp32) takes about 524 288 / 132 = 3 972
    rows (62 tiles), k_update_reduce then adds the 132 partials in fp32.  With every addend's rounding ~2^-24 of the
    running sum and random signs, the relative error of an element is about sqrt(3 972 + 132) * 2^-24 ~ 4e-6 of the sum
    of the addends' magnitudes; db_enc / db_heads run through per-thread fp32 sums of 62 * 16 rows, then shuffles and the
    same reduce, ~1e-6.  The 2e-5 stage bounds hold at this size with room to spare (observed below)."""
    rows, slabs, stride, n_act, seed, kw = UPDATE_CASES[name]
    with Peak():
        assert uu.case(rows, slabs, stride, n_act, seed, **kw)


def test_update_is_bitwise_reproducible_at_the_benchmark_layout():
    """The benchmark layout launched twice (minibatch 3 of 4, flush, advantages normalised in the kernel): bitwise-equal
    gradients and per-block sums of squares (the loss statistics are fp64 atomicAdds in no fixed order)."""
    dev = torch.device('cuda')
    torch.manual_seed(36)
    r_, g_, nm, mb, n_act = R_BENCH, 2, 4, 3, 4
    with Peak():
        xbuf = torch.randn(g_ * nm * r_, 128, device=dev)
        w_enc = torch.randn(128, 128, device=dev) * 0.1
        b_enc = torch.randn(128, device=dev) * 0.1
        w_cat = torch.zeros(8, 128, device=dev)
        w_cat[:n_act + 1] = torch.randn(n_act + 1, 128, device=dev) * 0.1
        b_cat = torch.zeros(8, device=dev)
        n = g_ * nm * r_
        act = torch.randint(0, n_act, (n,), device=dev)
        olp = torch.randn(n, device=dev) * 0.1 - 1.4
        adv, oval = torch.randn(n, device=dev), torch.randn(n, device=dev)
        an = torch.tensor([0.1, 0.9], device=dev)
        off, parts = uu.lib().pb_mlp_update_sumsq_offset(), uu.lib().pb_mlp_update_sumsq_parts()
        runs = []
        for _ in range(2):
            o = mb * r_
            gflat, _, _, _, _, ws = uu.fused(xbuf[o:], 128, r_, nm * r_, g_, w_enc, b_enc, w_cat, b_cat, act[o:], olp[o:],
                                             adv[o:], None, oval[o:], n_act, False, adv_norm=an, row_stride=nm * r_)
            torch.cuda.synchronize()
            runs.append((gflat, ws[off:off + 8 * parts].clone()))
        assert bool(torch.isfinite(runs[0][0]).all())
        assert torch.equal(runs[0][0].view(torch.int32), runs[1][0].view(torch.int32))
        assert torch.equal(runs[0][1], runs[1][1])


# ---- 2. train() on the benchmark workload, replayed ----------------------------------------------------------------------
def test_train_replays_at_the_benchmark_workload():
    """bench.py's workload (breakout, 16 384 x 128, bptt 16, 4 minibatches, 4 epochs, cuda_graph): the second train() is
    the captured one, on the plan ('mlp_fused', 'direct', 'whole'), and its 16 optimizer steps replay through
    test_gpu_experience.replay_direct_update with that test's bounds (parameters 1e-3 lr per step, second Adam moments
    1e-4 relative, equal step counts, the head matrix bitwise the pack of the parameters, the six losses), except the
    first Adam moments: 1e-3 of each one's maximum here.  The second moments (g^2 averaged, no cancellation) agree to
    1.3e-5, i.e. the two sides' gradients to ~5e-6 of their size; the first moments average gradients whose signs change
    from minibatch to minibatch, so they are smaller than the gradients they come from and the same differences are up
    to 4.1e-4 of them (b_val, b_enc, w_val).  Replaying with the device's own fp32 advantages instead of fp64 ones leaves
    2.3e-4: it is not the advantages' precision.  Parameters agree to 1.4e-6 (bound 4e-6)."""
    import bench
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    from test_gpu_experience import replay_direct_update
    n, h = 16384, 128
    cfg = bench.ppo_config(n, h, 'cuda')
    assert (cfg.batch_size, cfg.minibatch_size, cfg.bptt_horizon, cfg.update_epochs, cfg.cuda_graph) == \
        (n * h, n * h // 4, 16, 4, True)
    with Peak():
        vec = pvec.make(ocean.env_creator('breakout'), num_envs=n, backend=pvec.B200.options(exact_infos=False))
        torch.manual_seed(1)
        pol = cleanrl.Policy(models.Default(vec.driver_env, hidden_size=128), fused_sample=True, seed=1).cuda()
        data = clean_pufferl.create(cfg, vec, pol)
        norms = replay_direct_update(data, exp_avg_tol=1e-3)
        assert len(norms) == 16 and all(v == v for v in norms)
        assert data.train_graph_state == 2 and data.train_graph_replays == 1, data.msg
        plan = clean_pufferl.update_plan(data)
        assert (plan.engine, plan.form, plan.capture) == ('mlp_fused', 'direct', 'whole')
        clean_pufferl.close(data)


# ---- 3. the BPTT kernels at bench_lstm.py's minibatch --------------------------------------------------------------------
B_LSTM, T_LSTM = 32768, 16
SUBSETS = ((0, 64), (16384 - 64, 16384), (16384, 16384 + 64), (32768 - 64, 32768))    # segments [lo, hi)


def fp64_gemm_tn(a, b, chunk=1 << 15):
    """a^T b in fp64, K = rows, in chunks of rows."""
    acc = None
    for lo in range(0, a.shape[0], chunk):
        p = a[lo:lo + chunk].double().t() @ b[lo:lo + chunk].double()
        acc = p if acc is None else acc + p
    return acc


@pytest.mark.parametrize('hidden', [128, 256])
def test_bptt_kernels_at_the_bench_lstm_minibatch(hidden):
    """pb_lstm_bptt_forward / _backward on B = 32 768 segments x T = 16 (bench_lstm.py's minibatch), F = 128, 4 actions,
    with an initial state, NaN canaries past every output:
      * every output row finite, no canary written; the saved rows hold h_T, c_T (last step) and h0 (first step) bitwise;
      * on the first 64 segments, the last 64 and 64 on each side of segment 16 384: out, h_T, c_T and the saved h, c of
        every step against reference_step in fp64 (bounds of test_gpu_lstm_hidden256: 5e-4 after 16 steps), dz and dPre
        given the same dOut against fp64 autograd (reference_grads_h), 5e-3 of their maximum (TOL_GRAD); and every one of
        these rows bitwise equal to the kernels run on those 256 segments alone (a segment depends on its own rows only);
      * the ten weight gradients of _LSTMBPTTFunction.backward (the library GEMMs, _gemm_tn's split-K form at K = 524 288)
        against fp64 products of the kernel's own dz, saved rows, dPre and dOut: 2e-3 of each maximum for the TF32 GEMMs
        (each operand truncated or rounded to TF32, 2^-10 relative at most, so 2^-9 per product), 1e-5 for the fp32 sums."""
    from test_gpu_lstm_bptt import keep_relu_off_zero
    from test_gpu_lstm_hidden256 import (TOL_GRAD, TOL_SEQ, backward_kernel, forward_kernel, make_net,
                                         reference_grads_h)
    from test_gpu_policy_lstm import reference_step
    n_act, feats, bsz, steps, hid = 4, 128, B_LSTM, T_LSTM, hidden
    m = bsz * steps
    with Peak():
        net = make_net(feats, n_act, hidden=hid)
        gen = torch.Generator(device='cuda').manual_seed(hid)
        x = torch.rand(bsz, steps, feats, device='cuda', generator=gen) * 2 - 1
        keep_relu_off_zero(net, x)
        h0 = torch.randn(bsz, hid, device='cuda', generator=gen) * 0.5
        c0 = torch.randn(bsz, hid, device='cuda', generator=gen)
        dout = torch.randn(m, 8, device='cuda', generator=gen) / m ** 0.5
        dout[:, n_act + 1:] = 0

        # the weight gradients as train() forms them
        res = net.forward_packed_seq(x, (h0[None], c0[None]))
        assert res is not None
        net.zero_grad(set_to_none=True)
        res[0].backward(dout)
        del res
        got = {k: p.grad.clone() for k, p in list(net.policy.named_parameters()) + list(net.recurrent.named_parameters())}
        torch.cuda.empty_cache()

        # the whole minibatch through the kernels (forward_kernel / backward_kernel assert the canaries)
        out, hT, cT, saved = forward_kernel(net, x, h0, c0)
        dz, dpre = backward_kernel(net, dout, saved, c0, bsz, steps)
        for name, t in (('out', out), ('h_T', hT), ('c_T', cT), ('saved', saved), ('dz', dz), ('dPre', dpre)):
            assert bool(torch.isfinite(t).all()), f'{name}: a non-finite row'
        assert torch.equal(saved[steps - 1::steps, 7 * hid:], hT) and torch.equal(saved[steps - 1::steps, 6 * hid:7 * hid], cT)
        assert torch.equal(saved[0::steps, hid:2 * hid], h0)

        ok = True
        # stage check of the library GEMMs and sums of _LSTMBPTTFunction.backward
        w_gates = fp64_gemm_tn(dz, saved[:, :2 * hid])
        w_cat = fp64_gemm_tn(dout, saved[:, 7 * hid:])
        ref = {'weight_ih_l0': w_gates[:, :hid], 'weight_hh_l0': w_gates[:, hid:],
               'encoder.weight': fp64_gemm_tn(dpre, x.view(m, feats)),
               'decoder.weight': w_cat[:n_act], 'value_head.weight': w_cat[n_act:n_act + 1]}
        del w_gates
        for name, r in ref.items():
            ok &= uu.check(f'{name} (library GEMM) vs fp64', got[name], r, 2e-3)
        db_gates, db_cat = dz.sum(0, dtype=torch.float64), dout.sum(0, dtype=torch.float64)
        sums = {'bias_ih_l0': db_gates, 'bias_hh_l0': db_gates, 'encoder.bias': dpre.sum(0, dtype=torch.float64),
                'decoder.bias': db_cat[:n_act], 'value_head.bias': db_cat[n_act:n_act + 1]}
        for name, r in sums.items():
            ok &= uu.check(f'{name} (fp32 sum) vs fp64', got[name], r, 1e-5)

        # the subsets against fp64 and against the kernels run on them alone
        seg = torch.cat([torch.arange(lo, hi, device='cuda') for lo, hi in SUBSETS])
        rows = (seg[:, None] * steps + torch.arange(steps, device='cuda')).reshape(-1)
        xs, h0s, c0s, douts = x[seg], h0[seg], c0[seg], dout[rows]
        sub_saved = saved[rows].view(len(seg), steps, 8 * hid)
        errs = {'out': 0.0, 'h': 0.0, 'c': 0.0}
        with torch.no_grad():
            h, c = h0s.double(), c0s.double()
            sub_out = out[rows].view(len(seg), steps, -1)
            for t in range(steps):
                h, c, o = reference_step(net, xs[:, t], h, c)
                errs['out'] = max(errs['out'], float((sub_out[:, t].double() - o).abs().max()))
                errs['h'] = max(errs['h'], float((sub_saved[:, t, 7 * hid:].double() - h).abs().max()))
                errs['c'] = max(errs['c'], float((sub_saved[:, t, 6 * hid:7 * hid].double() - c).abs().max()))
        errs['h_T'] = float((hT[seg].double() - h).abs().max())
        errs['c_T'] = float((cT[seg].double() - c).abs().max())
        print(f'[bench-bptt] H={hid} B={bsz} T={steps} forward max err on the subsets',
              {k: f'{e:.2e}' for k, e in errs.items()}, flush=True)
        ok &= uu.claim(f'forward within TOL_SEQ = {TOL_SEQ}', all(e < TOL_SEQ for e in errs.values()))
        inner = {}
        reference_grads_h(net, xs, h0s, c0s, douts, inner)
        ok &= uu.check('dz on the subsets vs fp64 autograd', dz[rows], inner['dz'], TOL_GRAD)
        ok &= uu.check('dPre on the subsets vs fp64 autograd', dpre[rows], inner['dpre'], TOL_GRAD)
        s_out, s_hT, s_cT, s_saved = forward_kernel(net, xs, h0s, c0s)
        s_dz, s_dpre = backward_kernel(net, douts, s_saved, c0s, len(seg), steps)
        for name, a, b in (('out', out[rows], s_out), ('h_T', hT[seg], s_hT), ('c_T', cT[seg], s_cT),
                           ('saved', saved[rows], s_saved), ('dz', dz[rows], s_dz), ('dPre', dpre[rows], s_dpre)):
            ok &= uu.claim(f'{name} on the subsets bitwise the 256-segment launch', torch.equal(a, b))
        assert ok
