"""pb_mlp_tail_backward_ex (csrc/mlp_tail.cu), the backward of models.Default after the encoder GEMM: dPre, dW_heads,
db_enc and db_heads from one read of `hidden`, for R = 8, 16 and 32 head rows (Default.head_matrix) and 128 to 512 hidden
units, with dOut rows contiguous ([M, R]: the TMA-staged instance) or R + 4 floats apart (the strided one).

The helpers here are the ones the tail tests of test_gpu_default_heads16, test_gpu_default_heads32 and
test_gpu_default_hidden run on.  The tests below pin the bits: every instance computes a hidden column as one fmaf chain
over the head rows in k order, masks it, adds it to the column's accumulator row by row in the same warp order, and sums
the 8 warps of a CTA in warp order before k_reduce_partials.  The load mode, the slice width and zero-padded head rows
therefore change no output bit."""
import pytest
import torch

from pufferlib_b200 import _native

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
P = _native.ptr
HIDDEN = (128, 256, 384, 512)
BIG = 524288 + 17


def tail_inputs(m, hid, n_act, rows, seed, strided):
    torch.manual_seed(seed)
    hidden = torch.relu(torch.randn(m, hid, device=DEV))
    dout = torch.randn(m, rows, device=DEV) / max(m, 1) ** 0.5
    dout[:, n_act + 1:] = 0
    w = torch.randn(rows, hid, device=DEV)
    w[n_act + 1:] = 0
    if strided:            # rows head_rows + 4 floats apart: the strided instance
        wide = torch.zeros(m, rows + 4, device=DEV)
        wide[:, :rows] = dout
        dout = wide[:, :rows]
    return hidden, dout, w


def tail(dout, w, hidden, rows, ws=None, legacy=False):
    """dPre and the [R·H dW_heads | H db_enc | R db_heads] gradient row, both prefilled with NaN.  legacy: the 8-row
    entry point pb_mlp_tail_backward."""
    m, hid = hidden.shape
    lib = _native.lib()
    dpre = torch.full_like(hidden, float('nan'))
    grads = torch.full((rows * hid + hid + rows,), float('nan'), device=DEV)
    if legacy:
        assert rows == 8 and ws is None
        ws = torch.empty(lib.pb_mlp_tail_workspace_bytes(m, hid), dtype=torch.uint8, device=DEV)
        _native.check(lib.pb_mlp_tail_backward(P(dout), dout.stride(0), P(w), P(hidden), m, hid, P(dpre), P(grads), P(ws),
                                               ws.numel(), _native.stream_ptr()))
        return dpre, grads
    if ws is None:
        ws = torch.empty(lib.pb_mlp_tail_workspace_bytes_ex(m, hid, rows), dtype=torch.uint8, device=DEV)
    _native.check(lib.pb_mlp_tail_backward_ex(P(dout), dout.stride(0), P(w), P(hidden), m, hid, P(dpre), P(grads), P(ws),
                                              ws.numel(), rows, _native.stream_ptr()))
    return dpre, grads


def split(grads, rows, hid):
    """-> dW_heads [R, H], db_enc [H], db_heads [R]"""
    return grads[:rows * hid].view(rows, hid), grads[rows * hid:(rows + 1) * hid], grads[(rows + 1) * hid:]


def check_tail(dpre, grads, hidden, dout, w, rows, n_act):
    """Against fp64 torch: each output within 1e-5 of its maximum (all fp32 FMA); NaN (an entry never written) fails.
    The padding rows of dW_heads and db_heads are exactly 0."""
    h64, d64, w64 = hidden.double(), dout.double(), w.double()
    ref_dpre = (d64 @ w64) * (h64 > 0)
    dw, db_enc, db_heads = split(grads, rows, hidden.shape[1])
    refs = {'dpre': (dpre, ref_dpre), 'dW_heads': (dw, d64.t() @ h64), 'db_enc': (db_enc, ref_dpre.sum(0)),
            'db_heads': (db_heads, d64.sum(0))}
    for name, (got, ref) in refs.items():
        err = float((got.double() - ref).abs().max())
        assert err <= 1e-5 * float(ref.abs().max()) + 1e-30, (name, err, float(ref.abs().max()))
    assert float(dw[n_act + 1:].abs().sum()) == 0.0
    assert float(db_heads[n_act + 1:].abs().sum()) == 0.0


@pytest.mark.parametrize('m', [33, BIG])
@pytest.mark.parametrize('rows', [8, 16, 32])
@pytest.mark.parametrize('hid', HIDDEN)
def test_mlp_tail_load_modes_are_bitwise_equal(m, rows, hid):
    """The same dOut rows contiguous (TMA ring) and R + 4 floats apart (strided loads): torch.equal dPre and gradients."""
    out = []
    for strided in (False, True):
        hidden, dout, w = tail_inputs(m, hid, rows - 1, rows, m + hid + rows, strided)
        out.append(tail(dout, w, hidden, rows))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.parametrize('m', [513, BIG])
@pytest.mark.parametrize('rows', [8, 16, 32])
@pytest.mark.parametrize('hid', [256, 384, 512])
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_is_bitwise_its_128_column_runs(m, rows, hid, strided):
    """H = 256 to 512 against H = 128 runs on each 128-column run of the same rows (its columns of hidden and W_heads,
    the same dOut): torch.equal dPre columns, dW_heads columns and db_enc, and the same db_heads."""
    hidden, dout, w = tail_inputs(m, hid, rows - 1, rows, m + hid + rows, strided)
    dpre, grads = tail(dout, w, hidden, rows)
    dw, db_enc, db_heads = split(grads, rows, hid)
    for c in range(0, hid, 128):
        cols = slice(c, c + 128)
        dpre_c, grads_c = tail(dout, w[:, cols].contiguous(), hidden[:, cols].contiguous(), rows)
        dw_c, db_enc_c, db_heads_c = split(grads_c, rows, 128)
        assert torch.equal(dpre[:, cols], dpre_c), c
        assert torch.equal(dw[:, cols], dw_c) and torch.equal(db_enc[cols], db_enc_c), c
        assert torch.equal(db_heads, db_heads_c), c


@pytest.mark.parametrize('m', [513, BIG])
@pytest.mark.parametrize('hid', HIDDEN)
@pytest.mark.parametrize('strided', [False, True])
def test_mlp_tail_zero_padded_head_rows_are_bitwise_equal(m, hid, strided):
    """8 live head rows, zero-padded to 16 and to 32 rows (dOut columns and W_heads rows): torch.equal dPre and db_enc,
    the 8 live rows of dW_heads and db_heads equal to the 8-row run's, the padding rows exactly 0."""
    hidden, dout, w = tail_inputs(m, hid, 7, 8, m + hid, strided)
    dpre8, grads8 = tail(dout, w, hidden, 8)
    dw8, db_enc8, db_heads8 = split(grads8, 8, hid)
    for rows in (16, 32):
        dout_p = torch.zeros(m, rows + 4 * strided, device=DEV)[:, :rows]
        dout_p[:, :8] = dout
        w_p = torch.zeros(rows, hid, device=DEV)
        w_p[:8] = w
        dpre, grads = tail(dout_p, w_p, hidden, rows)
        dw, db_enc, db_heads = split(grads, rows, hid)
        assert torch.equal(dpre, dpre8) and torch.equal(db_enc, db_enc8), rows
        assert torch.equal(dw[:8], dw8) and torch.equal(db_heads[:8], db_heads8), rows
        assert bool((dw[8:] == 0).all()) and bool((db_heads[8:] == 0).all()), rows
