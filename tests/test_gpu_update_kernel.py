"""pb_mlp_update_fused through the C ABI (tests/util_update.py has the checks):
  * stage by stage: forward wgmma vs TF32-truncated fp64 math, dOut / statistics vs pb_ppo_loss on the kernel's own head
    outputs, dPre, and every gradient section vs fp64 products of the kernel's own dumps; then the same launch without dumps,
    and the refusal of a dPre output buffer (dW_enc is always formed in the kernel);
  * end to end: the six parameter gradients and the loss statistics vs a float64 autograd restatement whose encoder product
    takes TF32-truncated x and W_enc (so the TF32 rounding of the forward operands is checked by the stage-1 check only),
    the padding rows of the head gradients exactly 0, rows on both sides of the clip range;
  * the per-block sums of squares the reduce step leaves for pb_clip_adam_parts, after every launch, including a small
    launch on the workspace of a large one (test_sumsq_partials_after_a_larger_launch).
Shapes: one tile, a ragged tile count, more tiles than SMs, several slabs with gaps (the zero-copy minibatch layout), 1 / 4 / 7
actions, each with the benchmark's loss coefficients and with clip_vloss off and other coefficients
(test_fused_update_kernel_stages); the arguments train() passes on its zero-copy path -- arrival-order rows
(row_slab_stride = nm * R, pointer offset by one slab), returns formed in the kernel, the advantage normalisation applied in
the kernel, clip_vloss off, other loss coefficients -- for 1..7 actions, each on R = 288 (ragged tiles, 8 slabs, nm = 2) and
on R = 1024 (2 slabs, nm = 4) (test_fused_update_kernel_direct_path_arguments).  Reference of the math: reference
clean_pufferl.py:186-244 with the policy of pufferlib/models.py:12-62."""
import pytest
import torch

import util_update as uu

pytestmark = pytest.mark.gpu

SHAPES = [(128, 1, 128, 4, 1), (1000, 1, 1000, 4, 2), (148 * 128 * 2 + 77, 1, 148 * 128 * 2 + 77, 7, 3), (300, 2, 1000, 1, 4),
          (4096, 4, 16384, 4, 5)]
COEFS = {'bench': uu.CFG, 'alt': uu.CFG_ALT}                             # loss coefficients (util_update.CFG*)
DIRECT_SHAPES = {'r288': (288, 8, 2 * 288, 2), 'r1024': (1024, 2, 4 * 1024, 4)}   # slab_rows, n_slabs, slab_stride, nm
DIRECT_ARGS = {'as_train': dict(returns=False, adv_norm=True, cfg=uu.CFG),
               'as_train_no_vclip': dict(returns=False, adv_norm=True, cfg=uu.CFG_ALT),
               'no_old_values': dict(returns=True, old_values=False, cfg=uu.CFG_ALT)}


@pytest.mark.parametrize('coefs', list(COEFS))
@pytest.mark.parametrize('slab_rows,n_slabs,slab_stride,n_act,seed', SHAPES)
def test_fused_update_kernel_stages(slab_rows, n_slabs, slab_stride, n_act, seed, coefs):
    assert uu.case(slab_rows, n_slabs, slab_stride, n_act, seed, cfg=COEFS[coefs])


@pytest.mark.parametrize('layout', list(DIRECT_SHAPES))
@pytest.mark.parametrize('args', list(DIRECT_ARGS))
@pytest.mark.parametrize('n_act', range(1, 8))
def test_fused_update_kernel_direct_path_arguments(n_act, args, layout):
    slab_rows, n_slabs, slab_stride, nm = DIRECT_SHAPES[layout]
    assert uu.case(slab_rows, n_slabs, slab_stride, n_act, 100 + 10 * n_act + list(DIRECT_ARGS).index(args), nm=nm,
                   **DIRECT_ARGS[args])


def test_sumsq_partials_after_a_larger_launch():
    """One workspace through a launch on every SM, then launches on two CTAs and on a ragged slab layout: the sums of squares
    describe the latest gradient only."""
    ws = uu.workspace(torch.device('cuda'))
    assert uu.case(148 * 128 * 2 + 77, 1, 148 * 128 * 2 + 77, 7, 11, ws=ws)
    assert uu.case(128, 1, 128, 3, 12, ws=ws)
    assert uu.case(288, 8, 2 * 288, 5, 13, nm=2, returns=False, adv_norm=True, ws=ws)
