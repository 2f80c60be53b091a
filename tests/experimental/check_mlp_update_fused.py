"""Hardware check of the fused wgmma minibatch-update kernel (csrc/mlp_update.cu): the cases of tests/util_update.py (stage by
stage, end to end against float64 autograd, the sums of squares of the reduce step), then timing at the bench minibatch.  Not
collected by pytest (tests/test_gpu_update_kernel.py runs the same cases); run by hand on an H100 under a timeout:

    timeout 200 python tests/experimental/check_mlp_update_fused.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from util_update import case, fused, workspace  # noqa: E402

SHAPES = [(128, 1, 128, 4, 1), (1000, 1, 1000, 4, 2), (148 * 128 * 2 + 77, 1, 148 * 128 * 2 + 77, 7, 3), (300, 2, 1000, 1, 4),
          (4096, 4, 16384, 4, 5)]
DIRECT = [(288, 8, 2 * 288, 3, 6, 2), (1024, 2, 4 * 1024, 5, 7, 4)]     # ..., nm: the arrival-order rows of train()


def timing():
    dev = torch.device('cuda')
    m, n_act = 524288, 4
    torch.manual_seed(0)
    xbuf = torch.randn(4 * m, 128, device=dev)      # the 1 GiB rollout: two slabs of a minibatch are 2 M rows apart
    w_enc = torch.randn(128, 128, device=dev) * 0.1
    b_enc = torch.randn(128, device=dev) * 0.1
    w_cat = torch.zeros(8, 128, device=dev)
    w_cat[:n_act + 1] = torch.randn(n_act + 1, 128, device=dev) * 0.1
    b_cat = torch.zeros(8, device=dev)
    act = torch.randint(0, n_act, (m,), device=dev)
    olp = -torch.rand(m, device=dev) - 0.5
    adv, ret, oval = torch.randn(m, device=dev), torch.randn(m, device=dev), torch.randn(m, device=dev)
    ws = workspace(dev)
    for name, (rows, slabs, stride) in (('1 slab of 524288 rows', (m, 1, m)), ('2 slabs of 262144 rows', (m // 2, 2, 2 * m))):
        def fn(k):
            off = (k % 4) * (m // 2) if slabs == 2 else (k % 4) * m
            return fused(xbuf[off:], 128, rows, stride, slabs, w_enc, b_enc, w_cat, b_cat, act, olp, adv, ret, oval, n_act, False,
                         ws=ws)
        for k in range(3):
            fn(k)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(16):
            fn(k)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1000 / 16
        print(f'fused update, {name}: {us:8.1f} us / minibatch   x read at {m * 512 / us / 1e3:7.1f} GB/s', flush=True)


def main():
    ok = True
    for args in SHAPES:
        ok &= case(*args)
    for *args, nm in DIRECT:
        ok &= case(*args, nm=nm, returns=False, adv_norm=True)
    print('ALL OK' if ok else 'SOME MISMATCH', flush=True)
    timing()
    print('done')


if __name__ == '__main__':
    main()
