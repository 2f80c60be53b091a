"""pb_ppo_loss (one-pass PPO loss forward + analytic backward) vs the torch fp32 formulation of
reference clean_pufferl.py:202-238 differentiated by autograd.  Tolerance: 1e-5 relative on the loss and the
statistics, 1e-5 * max|grad| absolute on the gradients (fp32 expf / logf vs ATen's; no reordering beyond the sums)."""
import pytest
import torch

import pufferlib_b200
from pufferlib_b200 import clean_pufferl
from pufferlib_b200.frameworks import cleanrl

pytestmark = pytest.mark.gpu


def reference_loss(logits, value, actions, old_lp, adv, ret, old_v, cfg):
    _, newlogprob, entropy = cleanrl.sample_logits(logits, actions)
    logratio = newlogprob - old_lp
    ratio = logratio.exp()
    old_kl = (-logratio).mean()
    kl = ((ratio - 1) - logratio).mean()
    clipfrac = ((ratio - 1.0).abs() > cfg.clip_coef).float().mean()
    pg = torch.max(-adv * ratio, -adv * torch.clamp(ratio, 1 - cfg.clip_coef, 1 + cfg.clip_coef)).mean()
    nv = value.view(-1)
    if cfg.clip_vloss:
        vc = old_v + torch.clamp(nv - old_v, -cfg.vf_clip_coef, cfg.vf_clip_coef)
        vl = 0.5 * torch.max((nv - ret) ** 2, (vc - ret) ** 2).mean()
    else:
        vl = 0.5 * ((nv - ret) ** 2).mean()
    ent = entropy.mean()
    loss = pg - cfg.ent_coef * ent + vl * cfg.vf_coef
    return loss, torch.stack([pg, vl, ent, old_kl, kl, clipfrac]).detach()


@pytest.mark.parametrize('m,n_act', [(1, 4), (1000, 4), (4097, 6), (524288, 4), (333, 18), (4097, 1), (4097, 32),
                                     (1, 32)])
@pytest.mark.parametrize('clip_vloss', [True, False])
def test_ppo_loss_matches_torch_autograd(m, n_act, clip_vloss):
    dev = torch.device('cuda')
    torch.manual_seed(m + n_act)
    cfg = pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=clip_vloss, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    base = torch.randn(m, 8 if n_act < 8 else n_act + 3, device=dev)            # strided heads, like the merged GEMM
    logits0 = base[:, :n_act]
    value0 = base[:, n_act:n_act + 1] if base.shape[1] > n_act else torch.randn(m, 1, device=dev)
    actions = torch.randint(0, n_act, (m,), device=dev)
    with torch.no_grad():
        _, nlp, _ = cleanrl.sample_logits(logits0, actions)
    old_lp = nlp + 0.2 * torch.randn(m, device=dev)
    old_lp[::3] = nlp[::3]                      # exact ties: ratio == 1 (inside the clip range, pg1 == pg2)
    adv = torch.randn(m, device=dev)
    ret = torch.randn(m, device=dev)
    old_v = value0.detach().view(-1) + 0.15 * torch.randn(m, device=dev)

    la, va = logits0.detach().clone().requires_grad_(True), value0.detach().clone().requires_grad_(True)
    loss_ref, st_ref = reference_loss(la, va, actions, old_lp, adv, ret, old_v, cfg)
    loss_ref.backward()

    lb, vb = logits0.detach().clone().requires_grad_(True), value0.detach().clone().requires_grad_(True)
    loss, st = clean_pufferl.fused_ppo_loss(lb, vb, actions, old_lp, adv, ret, old_v, cfg)
    loss.backward()

    assert torch.allclose(loss, loss_ref, rtol=1e-5, atol=1e-6)
    assert torch.allclose(st, st_ref, rtol=1e-5, atol=1e-6)
    for g, gr in ((lb.grad, la.grad), (vb.grad, va.grad)):
        assert g.shape == gr.shape
        assert float((g - gr).abs().max()) <= 1e-5 * float(gr.abs().max()) + 1e-10


def test_ppo_loss_through_strided_views_and_scaling():
    """Gradients flow back through slices of one merged-head GEMM output, and backward scales with grad_output."""
    dev = torch.device('cuda')
    torch.manual_seed(0)
    cfg = pufferlib_b200.namespace(clip_coef=0.2, clip_vloss=True, vf_clip_coef=0.2, vf_coef=1.0, ent_coef=0.0)
    m, n_act = 257, 4
    out = torch.randn(m, 8, device=dev, requires_grad=True)
    actions = torch.randint(0, n_act, (m,), device=dev)
    old_lp, adv, ret, old_v = (torch.randn(m, device=dev) * 0.1 - 1.4, torch.randn(m, device=dev),
                               torch.randn(m, device=dev), torch.randn(m, device=dev))
    loss, _ = clean_pufferl.fused_ppo_loss(out[:, :n_act], out[:, n_act:n_act + 1], actions, old_lp, adv, ret, old_v, cfg)
    (3.0 * loss).backward()
    out2 = out.detach().clone().requires_grad_(True)
    ref, _ = reference_loss(out2[:, :n_act], out2[:, n_act:n_act + 1], actions, old_lp, adv, ret, old_v, cfg)
    (3.0 * ref).backward()
    assert torch.allclose(out.grad, out2.grad, rtol=1e-4, atol=1e-7)
    assert float(out.grad[:, n_act + 1:].abs().sum()) == 0.0


def test_default_mlp_fast_path_matches_plain_modules():
    """models.Default fast path (fused GEMM epilogues + pb_mlp_tail_backward) vs the plain nn.Linear / relu composition:
    same outputs and the same parameter gradients (TF32 tensor-core GEMMs on both sides -> ~1e-3 relative)."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import models
    from pufferlib_b200.environments import ocean
    dev = torch.device('cuda')
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=4, backend=pvec.B200)
    torch.manual_seed(0)
    net = models.Default(vec.driver_env).to(dev)
    for m in (1, 37, 4096, 70001):
        x = torch.randn(m, 128, device=dev)
        g_logits, g_value = torch.randn(m, 4, device=dev), torch.randn(m, 1, device=dev)
        grads = []
        for fast in (True, False):
            net.fast_path = fast
            net.zero_grad()
            logits, value = net(x)
            ((logits * g_logits).sum() + (value * g_value).sum()).backward()
            grads.append((logits.detach(), value.detach(), [p.grad.clone() for p in net.parameters()]))
        (l1, v1, g1), (l0, v0, g0) = grads
        assert torch.allclose(l1, l0, rtol=2e-3, atol=2e-3) and torch.allclose(v1, v0, rtol=2e-3, atol=2e-3)
        for a, b in zip(g1, g0):
            scale = float(b.abs().max()) + 1e-6
            assert float((a - b).abs().max()) <= 5e-3 * scale, (m, float((a - b).abs().max()), scale)
    vec.close()


@pytest.mark.parametrize('m,n_act', [(1, 4), (4097, 6), (100000, 7)])
def test_ppo_loss_packed_rows(m, n_act):
    """Packed [M, 8] rows (n_act logits | value | zero pad): 128-bit row accesses, ONE [M, 8] gradient back."""
    dev = torch.device('cuda')
    torch.manual_seed(m)
    cfg = pufferlib_b200.namespace(clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01)
    out0 = torch.randn(m, 8, device=dev)
    out0[:, n_act + 1:] = 0
    actions = torch.randint(0, n_act, (m,), device=dev)
    old_lp, adv, ret = -torch.rand(m, device=dev) - 1, torch.randn(m, device=dev), torch.randn(m, device=dev)
    old_v = out0[:, n_act] + 0.15 * torch.randn(m, device=dev)
    a = out0.clone().requires_grad_(True)
    loss, st = clean_pufferl.fused_ppo_loss_packed(a, n_act, actions, old_lp, adv, ret, old_v, cfg)
    loss.backward()
    b = out0.clone().requires_grad_(True)
    ref, st_ref = reference_loss(b[:, :n_act], b[:, n_act:n_act + 1], actions, old_lp, adv, ret, old_v, cfg)
    ref.backward()
    assert torch.allclose(loss, ref, rtol=1e-5, atol=1e-6) and torch.allclose(st, st_ref, rtol=1e-5, atol=1e-6)
    assert float((a.grad - b.grad).abs().max()) <= 1e-5 * float(b.grad.abs().max()) + 1e-10
    assert float(a.grad[:, n_act + 1:].abs().sum()) == 0.0


@pytest.mark.parametrize('m', [1, 100, 128, 16384, 20001])
def test_fused_policy_step_matches_torch_policy(m):
    """pb_policy_mlp_sample (encoder + ReLU + heads + sampling in one mma.sync kernel) vs the torch modules: logprob of
    the sampled actions, entropy and value agree to TF32 accuracy (2e-3), actions are valid and follow the softmax."""
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import models
    from pufferlib_b200.environments import ocean
    dev = torch.device('cuda')
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=4, backend=pvec.B200)
    torch.manual_seed(1)
    net = models.Default(vec.driver_env).to(dev)
    with torch.no_grad():
        net.decoder.weight.mul_(30.0)            # the 0.01-std init gives near-uniform logits: make them informative
    pol = cleanrl.Policy(net, fused_sample=True, seed=5).to(dev)
    x = torch.randn(m, 128, device=dev)
    vr, lr = torch.zeros(m, device=dev), torch.zeros(m, device=dev)
    ar = torch.full((m,), -1, dtype=torch.int64, device=dev)
    with torch.no_grad():
        a, lp, ent, v = pol(x, out=(vr, lr, ar))
        assert a.data_ptr() == ar.data_ptr() and v.data_ptr() == vr.data_ptr()
        net.fast_path = False
        _, ref_lp, ref_ent, ref_v = pol(x, action=ar)             # plain torch modules, same actions
        logits, _ = net(x)
        net.fast_path = True
    assert int(ar.min()) >= 0 and int(ar.max()) < 4
    assert torch.allclose(lr, ref_lp, atol=3e-3), float((lr - ref_lp).abs().max())
    assert torch.allclose(ent, ref_ent, atol=3e-3) and torch.allclose(vr, ref_v.flatten(), atol=3e-3)
    if m >= 16384:
        freq = torch.bincount(ar, minlength=4).float() / m
        expect = torch.softmax(logits, -1).mean(0)
        assert float((freq - expect).abs().max()) < 0.02
    # the kernel's last CTA advances the device draw counter: one per call, and the next call draws fresh numbers
    assert int(pol._counter.item()) == 1 and int(pol._ticket.item()) == 0
    with torch.no_grad():
        a2, _, _, _ = pol(x)
    assert int(pol._counter.item()) == 2 and int(pol._ticket.item()) == 0
    if m >= 16384:
        assert 0.3 < float((a2 != ar).float().mean()) < 0.95
    vec.close()
