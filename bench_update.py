#!/usr/bin/env python
"""bench_update.py -- the fused minibatch update (pb_mlp_update_fused, csrc/mlp_update.cu) at the size bench.py runs it.

    python bench_update.py [--launches N] [--out DIR] [--parent-src DIR]

Builds bench.py's trainer (make_b200 / ppo_config: breakout, 16 384 envs x 128 steps, 4 minibatches), fills the rollout
with one evaluate(), and launches pb_mlp_update_fused on the zero-copy slab views of the four minibatches the way train()
passes them (x [G, R, 128] slab views of the rollout, R rows per slab, slab stride nm * R).  Prints one JSON line with
  * `update`: µs per launch (CUDA events over --launches back-to-back launches rotating over the four minibatches, median
    of 5 windows), and the fractions of the two bounds of one launch: HBM (x once + 28 B of per-row scalars per row, at the
    H100 SXM data sheet's 3.35 TB/s) and tensor core (forward and dW_enc products, 2 x 2 x M x 128 x 128 flop, at the data
    sheet's 495 TFLOP/s dense TF32); `bound` names the larger;
  * `phases`: the kernel built again with -DPB_UPDATE_PHASES into DIR (a library of its own, next to a small stub for
    the few host helpers it needs): one lane per warpgroup stamps clock64() at each phase boundary of the first tiles it
    handles; median SM cycles of every phase over all CTAs (the first tile of each warpgroup left out);
  * with --parent-src (a copy of another revision's pufferlib_b200/csrc and include, e.g. the parent commit's), that
    revision's kernel built the same way: one seeded bench-size minibatch through both (gradient max error over max |ref|,
    loss statistics), launch times alternated, and its phases when its sources carry the same instrumentation.
The card's name and power limit go with the numbers.  Writes nothing to the tree (DIR defaults to a temporary directory)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import tempfile
import types

import numpy as np
import torch

from bench import gpu_info, make_b200

HERE = os.path.dirname(os.path.abspath(__file__))
HBM_PEAK = 3.35e12        # H100 SXM data sheet, bytes/s
TF32_PEAK = 495e12        # H100 SXM data sheet, dense TF32 flop/s
NDW, TAIL = 128 * 128, 8 * 128 + 128 + 8

# the host helpers csrc/mlp_update.cu calls (csrc/abi.cu has them, next to everything else of the library)
STUB = r'''
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
unsigned long long g_pb_launches = 0;
static char g_err[512];
void pb_set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap); }
extern "C" const char* pb_phase_lib_error(void) { return g_err; }
int pb_num_sms() { int d = 0, n = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); return n; }
'''


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=100, help='launches per timed window (5 windows)')
    ap.add_argument('--out', default=None, help='directory for the instrumented libraries (default: a temporary one)')
    ap.add_argument('--parent-src', default=None, help="another revision's tree (pufferlib_b200/csrc + include) to compare")
    return ap.parse_args()


def nvcc():
    return os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')


def build_lib(src_root, out_dir, phases):
    """csrc/mlp_update.cu of `src_root` (+ the host-helper stub) -> out_dir/libupdate.so."""
    os.makedirs(out_dir, exist_ok=True)
    stub = os.path.join(out_dir, 'stub.cu')
    with open(stub, 'w') as f:
        f.write(STUB)
    csrc = os.path.join(src_root, 'pufferlib_b200', 'csrc')
    so = os.path.join(out_dir, 'libupdate.so')
    cmd = [nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xcompiler', '-fPIC', '-shared',
           '-I', os.path.join(src_root, 'include'), '-I', csrc] + (['-DPB_UPDATE_PHASES'] if phases else []) + [
           os.path.join(csrc, 'mlp_update.cu'), stub, '-o', so, '-lcudart']
    subprocess.check_call(cmd)
    lib = C.CDLL(so)
    from pufferlib_b200 import _native
    lib.pb_mlp_update_fused.restype = C.c_int
    lib.pb_mlp_update_fused.argtypes = _native.lib().pb_mlp_update_fused.argtypes
    lib.pb_mlp_update_workspace_bytes.restype = C.c_size_t
    lib.pb_phase_lib_error.restype = C.c_char_p
    return lib


def check(lib, rc):
    if rc != 0:
        raise RuntimeError(lib.pb_phase_lib_error().decode())


class Workload:
    """The four minibatches of one bench.py step as train() hands them to pb_mlp_update_fused."""

    def __init__(self):
        from pufferlib_b200 import clean_pufferl as cp
        args = types.SimpleNamespace(num_envs=16384, horizon=128, env='breakout', hidden=128, minibatches=4, epochs=4)
        self.data, _ = make_b200(args, 0, 1, False, True)
        cp.evaluate(self.data)
        torch.cuda.synchronize()
        n, h, nm = args.num_envs, args.horizon, args.minibatches
        exp = self.data.experience
        g_, r_ = cp.slab_layout(n, h, nm, 16)
        self.g, self.r, self.nm, self.mb = g_, r_, nm, n * h // nm
        self.xs = [exp.obs.view(g_, nm, r_, 128)[:, k] for k in range(nm)]
        self.n_act = self.data.vecenv.single_action_space.n
        model = self.data.policy.policy
        self.w_enc, self.b_enc = model.encoder.weight.detach(), model.encoder.bias.detach()
        self.w_cat, self.b_cat = [t.detach() for t in model.head_matrix()]
        gen = torch.Generator(device='cuda').manual_seed(7)
        mb = self.mb
        self.acts = torch.randint(0, self.n_act, (mb,), device='cuda', generator=gen)
        self.olp = torch.randn(mb, device='cuda', generator=gen) * 0.1 - np.log(self.n_act)
        self.adv = torch.randn(mb, device='cuda', generator=gen)
        self.ret = torch.randn(mb, device='cuda', generator=gen)
        self.oval = torch.randn(mb, device='cuda', generator=gen)

    def launcher(self, lib):
        ws = torch.empty(lib.pb_mlp_update_workspace_bytes(), dtype=torch.uint8, device='cuda')
        gfl = torch.empty(NDW + TAIL, device='cuda')
        st = torch.zeros(8, dtype=torch.float64, device='cuda')
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)

        def launch(i=0):
            x = self.xs[i % self.nm]
            rc = lib.pb_mlp_update_fused(
                p(x), 128, self.r, x.stride(0) // 128 if self.g > 1 else self.r, self.g, p(self.w_enc), p(self.b_enc),
                p(self.w_cat), p(self.b_cat), p(self.acts), p(self.olp), p(self.adv), p(self.ret), p(self.oval), None, self.r,
                self.n_act, C.c_float(0.1), 1, C.c_float(0.1), C.c_float(0.5), C.c_float(0.01), p(gfl), p(st), p(ws),
                ws.numel(), None, None, None, None, s)
            if rc != 0:
                raise RuntimeError(f'pb_mlp_update_fused failed ({rc})')
        return launch, gfl, st


def alternate(fns, reps, windows=5):
    """{name: median over `windows` of the per-launch time (s) of `reps` back-to-back launches}, names alternated."""
    for f in fns.values():
        for i in range(4):
            f(i)
    times = {k: [] for k in fns}
    for _ in range(windows):
        for k, f in fns.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(reps):
                f(i)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e-3 / reps)
    return {k: float(np.median(v)) for k, v in times.items()}


def bounds(t, m):
    t_hbm = m * (512 + 28) / HBM_PEAK
    t_tc = 2 * 2 * m * 128 * 128 / TF32_PEAK
    return dict(us=round(t * 1e6, 2), hbm_bound_us=round(t_hbm * 1e6, 1), tf32_bound_us=round(t_tc * 1e6, 1),
                frac_of_hbm_bound=round(t_hbm / t, 3), frac_of_tf32_bound=round(t_tc / t, 3),
                bound='hbm' if t_hbm >= t_tc else 'tf32')


def phases(lib, wl):
    """Median cycles of each phase of each warpgroup: stamp i to stamp i + 1, and the last stamp to the next tile's first;
    the first sampled tile of every warpgroup is left out (W_enc and the first x tiles arriving)."""
    tiles, nph = C.c_int32(), C.c_int32()
    n_wg = lib.pb_mlp_update_phase_layout(C.byref(tiles), C.byref(nph))
    lib.pb_mlp_update_phase_names.restype = C.c_char_p
    names = [x.split(',') for x in lib.pb_mlp_update_phase_names().decode().split(';')]    # one list per warpgroup
    grid = torch.cuda.get_device_properties(0).multi_processor_count
    buf = torch.zeros(grid * n_wg * tiles.value * nph.value, dtype=torch.int64, device='cuda')
    launch, _, _ = wl.launcher(lib)
    launch(0)
    check(lib, lib.pb_mlp_update_set_phase_buffer(C.c_void_p(buf.data_ptr())))
    launch(0)
    torch.cuda.synchronize()
    check(lib, lib.pb_mlp_update_set_phase_buffer(None))
    a = buf.view(grid, n_wg, tiles.value, nph.value).cpu().numpy().astype(np.float64)
    out = {}
    for w in range(n_wg):
        role = names[w]
        k = len(role) - 1
        st = a[:, w, :, :k + 1]
        ok = (st > 0).all(2)
        pair = ok[:, 1:] & ok[:, :-1]
        rows = {}
        for i in range(k):
            d, v = (st[:, :, i + 1] - st[:, :, i])[:, 1:], ok[:, 1:]
            rows[role[i]] = float(np.median(d[v])) if v.any() else None
        d = st[:, 1:, 0] - st[:, :-1, k]
        rows[role[k]] = float(np.median(d[pair])) if pair.any() else None
        d = st[:, 1:, 0] - st[:, :-1, 0]
        rows['whole tile'] = float(np.median(d[pair])) if pair.any() else None
        out[f'warpgroup{w}'] = rows
    return dict(unit='SM cycles, median over CTAs and sampled tiles', **out)


def main():
    args = parse_args()
    torch.cuda.set_device(0)
    from pufferlib_b200 import _native
    out_dir = args.out or tempfile.mkdtemp(prefix='bench_update_')
    wl = Workload()
    line = dict(gpu=gpu_info(0), rows_per_minibatch=wl.mb, slabs=wl.g, slab_rows=wl.r, n_act=wl.n_act,
                launches_per_window=args.launches, windows=5, statistic='median')
    libs = {'new': _native.lib()}
    if args.parent_src:
        libs['parent'] = build_lib(args.parent_src, os.path.join(out_dir, 'parent'), False)
    fns = {}
    for k, lib in libs.items():
        fns[k] = wl.launcher(lib)[0]
    t = alternate(fns, args.launches)
    line['update'] = {k: bounds(v, wl.mb) for k, v in t.items()}
    if 'parent' in t:
        line['update']['speedup'] = round(t['parent'] / t['new'], 3)
        res = {}
        for k, lib in libs.items():
            launch, gfl, st = wl.launcher(lib)
            launch(0)
            torch.cuda.synchronize()
            res[k] = (gfl.double().clone(), st.clone())
        (g_new, s_new), (g_ref, s_ref) = res['new'], res['parent']
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max())  # noqa: E731
        line['same_results'] = dict(gflat_rel=rel(g_new, g_ref), stats_rel=rel(s_new[:6], s_ref[:6]),
                                    gflat_ok=rel(g_new, g_ref) <= 2e-5, stats_ok=rel(s_new[:6], s_ref[:6]) <= 2e-3)
    lib_ph = build_lib(HERE, os.path.join(out_dir, 'phases'), True)
    line['phases'] = {'new': phases(lib_ph, wl)}
    if args.parent_src:
        lib_pp = build_lib(args.parent_src, os.path.join(out_dir, 'parent_phases'), True)
        if hasattr(lib_pp, 'pb_mlp_update_phase_names'):
            line['phases']['parent'] = phases(lib_pp, wl)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
