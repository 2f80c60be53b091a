"""pb_mlp_update_fused at the boundaries of its tile loop (csrc/mlp_update.cu: one CTA per SM looping over 64-row tiles,
a ring of NSTAGE x tiles), with the stage-by-stage checks of tests/util_update.py:
  * an odd number of tiles on every CTA;
  * slabs shorter than one tile (every tile ragged) and slabs whose row count is not a multiple of the tile;
  * enough tiles per CTA that every x stage goes round several times;
each with the benchmark's loss coefficients and with clip_vloss off and other coefficients (util_update.CFG_ALT); and that the same launch twice gives a bitwise-equal gradient and the same per-block sums of squares (the loss statistics are
left out: their fp64 atomicAdds land in no fixed order)."""
import pytest
import torch

import util_update as uu

pytestmark = pytest.mark.gpu


def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def schedule_shapes():
    s = n_sms()
    return {'odd_tiles_per_cta': (3 * 64 * s, 1, 3 * 64 * s, 5, 21),
            'slabs_shorter_than_a_tile': (20, 3, 40, 4, 22),
            'ragged_slabs': (100, 5, 160, 7, 23),
            'many_tiles_per_cta': (8192, 8, 8192, 3, 24)}


@pytest.mark.parametrize('coefs', ['bench', 'alt'])
@pytest.mark.parametrize('shape', ['odd_tiles_per_cta', 'slabs_shorter_than_a_tile', 'ragged_slabs', 'many_tiles_per_cta'])
def test_update_schedule_boundaries(shape, coefs):
    assert uu.case(*schedule_shapes()[shape], cfg=uu.CFG if coefs == 'bench' else uu.CFG_ALT)


@pytest.mark.parametrize('slab_rows,n_slabs,slab_stride', [(4096 * 4 + 17, 4, 4096 * 8), (96, 1, 96)])
def test_update_is_bitwise_reproducible(slab_rows, n_slabs, slab_stride):
    dev = torch.device('cuda')
    torch.manual_seed(5)
    n_act = 6
    m = slab_rows * n_slabs
    xbuf = torch.randn((n_slabs - 1) * slab_stride + slab_rows, 128, device=dev)
    w_enc = torch.randn(128, 128, device=dev) * 0.1
    b_enc = torch.randn(128, device=dev) * 0.1
    w_cat = torch.zeros(8, 128, device=dev)
    w_cat[:n_act + 1] = torch.randn(n_act + 1, 128, device=dev) * 0.1
    b_cat = torch.zeros(8, device=dev)
    act = torch.randint(0, n_act, (m,), device=dev)
    olp = torch.randn(m, device=dev) * 0.1 - 1.8
    adv, ret, oval = torch.randn(m, device=dev), torch.randn(m, device=dev), torch.randn(m, device=dev)
    off, n = uu.lib().pb_mlp_update_sumsq_offset(), uu.lib().pb_mlp_update_sumsq_parts()
    runs = []
    for _ in range(2):
        gflat, _, _, _, _, ws = uu.fused(xbuf, 128, slab_rows, slab_stride, n_slabs, w_enc, b_enc, w_cat, b_cat, act, olp, adv,
                                         ret, oval, n_act, False)
        torch.cuda.synchronize()
        runs.append((gflat, ws[off:off + 8 * n].clone()))
    assert bool(torch.isfinite(runs[0][0]).all())
    assert torch.equal(runs[0][0].view(torch.int32), runs[1][0].view(torch.int32))
    assert torch.equal(runs[0][1], runs[1][1])
