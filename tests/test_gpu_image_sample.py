"""pb_image_pack (TMA frame-stack pack) vs numpy, and the fused sampling epilogue vs the torch formulation of
pufferlib/frameworks/cleanrl.py:25-47."""
import ctypes as C

import numpy as np
import pytest
import torch

from pufferlib_b200 import _native
from pufferlib_b200.frameworks import cleanrl

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('n,stack,frame', [(1, 4, 7056), (37, 4, 7056), (1000, 4, 7056), (64, 2, 1024), (9, 1, 4096)])
def test_image_pack_vs_numpy(n, stack, frame):
    dev = torch.device('cuda')
    g = torch.Generator().manual_seed(n)
    new = torch.randint(0, 256, (n, frame), dtype=torch.uint8, generator=g).to(dev)
    prev = torch.randint(0, 256, (n, stack, frame), dtype=torch.uint8, generator=g).to(dev)
    reset = (torch.rand(n, generator=g) < 0.3).to(torch.uint8).to(dev)
    out = torch.zeros(n, stack, frame, dtype=torch.uint8, device=dev)
    lib = _native.lib()
    _native.check(lib.pb_image_pack(_native.ptr(new), frame, _native.ptr(prev), stack * frame, _native.ptr(out),
                                    stack * frame, _native.ptr(reset), n, frame, stack, _native.stream_ptr()))
    ref = torch.cat([prev[:, 1:], new[:, None]], dim=1)
    ref = torch.where(reset.bool()[:, None, None], new[:, None].expand(n, stack, frame), ref)
    assert torch.equal(out, ref)
    # in place (prev == out) is allowed: the old frames are staged in shared memory before the store
    buf = prev.clone()
    _native.check(lib.pb_image_pack(_native.ptr(new), frame, _native.ptr(buf), stack * frame, _native.ptr(buf),
                                    stack * frame, None, n, frame, stack, _native.stream_ptr()))
    assert torch.equal(buf, torch.cat([prev[:, 1:], new[:, None]], dim=1))


def test_image_pack_rejects_misaligned():
    from pufferlib_b200.exceptions import APIUsageError
    x = torch.zeros(4, 4, 100, dtype=torch.uint8, device='cuda')
    with pytest.raises(APIUsageError):
        _native.check(_native.lib().pb_image_pack(_native.ptr(x), 100, _native.ptr(x), 400, _native.ptr(x), 400, None, 4,
                                                  100, 4, _native.stream_ptr()))


@pytest.mark.parametrize('n,n_act', [(1, 4), (1000, 8), (16384, 4), (4096, 6), (333, 18)])
def test_sample_logits_logprob_entropy_match_torch(n, n_act):
    dev = torch.device('cuda')
    torch.manual_seed(n + n_act)
    logits = (torch.randn(n, n_act, device=dev) * 2).contiguous()
    actions = torch.empty(n, dtype=torch.int64, device=dev)
    logprob = torch.empty(n, device=dev)
    ent = torch.empty(n, device=dev)
    value = torch.randn(n, device=dev)
    vr, lr, ar = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, dtype=torch.int64, device=dev)
    _native.check(_native.lib().pb_sample_logits(
        _native.ptr(logits), n_act, n, n_act, C.c_uint64(7), C.c_uint64(3), None, _native.ptr(actions), _native.ptr(logprob),
        _native.ptr(ent), _native.ptr(value), 1, _native.ptr(vr), _native.ptr(lr), _native.ptr(ar), _native.stream_ptr()))
    assert int(actions.min()) >= 0 and int(actions.max()) < n_act
    _, ref_lp, ref_ent = cleanrl.sample_logits(logits, action=actions)      # torch formulation, same actions
    assert torch.allclose(logprob, ref_lp, rtol=1e-5, atol=1e-5)
    assert torch.allclose(ent, ref_ent, rtol=1e-5, atol=1e-5)
    assert torch.equal(ar, actions) and torch.equal(lr, logprob) and torch.equal(vr, value)


def test_fused_policy_writes_rollout_rows_and_strided_heads():
    """cleanrl.Policy(fused_sample=True): both heads come out of one GEMM (strided logits / value) and the epilogue
    writes value / logprob / action straight into the given rollout rows."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import models
    from pufferlib_b200.environments import ocean
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=257, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=3).cuda()
    obs = torch.randn(257, 128, device='cuda')
    vr, lr = torch.zeros(257, device='cuda'), torch.zeros(257, device='cuda')
    ar = torch.full((257,), -1, dtype=torch.int64, device='cuda')
    with torch.no_grad():
        a, lp, ent, v = pol(obs, out=(vr, lr, ar))
        assert a.data_ptr() == ar.data_ptr() and lp.data_ptr() == lr.data_ptr() and v.data_ptr() == vr.data_ptr()
        _, ref_lp, ref_ent, ref_v = pol(obs, action=ar)           # torch formulation on the same actions
    assert int(ar.min()) >= 0 and int(ar.max()) < 4
    # the fused step evaluates the MLP with mma.sync TF32 tiles, the torch path with cuBLAS TF32: ~1e-3 agreement
    assert torch.allclose(lr, ref_lp, atol=3e-3) and torch.allclose(ent, ref_ent, atol=3e-3)
    assert torch.allclose(vr, ref_v.flatten(), atol=3e-3)
    # two heads in one GEMM == two separate Linear layers (TF32 tensor-core GEMMs: ~1e-3 relative)
    hid = torch.relu(pol.policy.encoder(obs))
    assert torch.allclose(pol.policy.decode_actions(hid, None)[0], pol.policy.decoder(hid), atol=5e-3)
    assert torch.allclose(pol.policy.decode_actions(hid, None)[1], pol.policy.value_head(hid), atol=5e-3)
    vec.close()
