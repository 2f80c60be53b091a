"""The PPO loss kernels where the loss changes branch and at the logits real policies produce, against fp64 autograd of
tests/test_gpu_ppo_loss.reference_loss (cleanrl.sample_logits / cleanrl.entropy), and the fp32 torch formulation where
parity with the reference trainer is the point.

* pb_ppo_loss (csrc/ppo_loss.cu) through its four instances: W = 0 on strided column views (the 'model' engine), and the
  packed [M, 8], [M, 16] and [M, 32] rows (n_act <= 7, <= 15, <= 31), at M = 1, 255, 256, 257 (the 256-row block's
  edges) and 65 537 (a multi-block launch):
  - masked actions (-inf, finfo(float32).min and -1e30 logits): every output finite, masked-column gradients exactly 0;
  - logits sharing a large offset C: the probabilities are renormalised, so the entropy is cleanrl.entropy's;
  - rows exactly on the clamp edges and on the tie of the two value losses, built from dyadic values or from the
    device's own exp so that both sides see the same fp32 numbers: gradients follow the ATen rules (clamp passes the
    gradient at its bounds; maximum splits it at ties).
* The loss epilogue of k_mlp_update (csrc/mlp_update.cu) at the same edges, with W_cat = 0 so the logits are b_cat.
* train() with a policy that masks unavailable bandit arms, and with a 40-action head (past pb_ppo_loss's 32)."""
import numpy as np
import pytest
import torch

import pufferlib_b200
import pufferlib_b200.vector as pvec
import util_update as uu
from pufferlib_b200 import clean_pufferl
from pufferlib_b200.environments import ocean
from pufferlib_b200.frameworks import cleanrl
from test_gpu_experience import make_config
from test_gpu_ppo_loss import reference_loss

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
MS = [1, 255, 256, 257, 65537]
LAYOUTS = ['strided', 'packed']
FMIN = float(torch.finfo(torch.float32).min)


def loss_cfg(clip=0.1, vclip=0.1, clip_vloss=True):
    return pufferlib_b200.namespace(clip_coef=clip, clip_vloss=clip_vloss, vf_clip_coef=vclip, vf_coef=0.5, ent_coef=0.01)


def packed_width(n_act):
    return 8 if n_act <= 7 else 16 if n_act <= 15 else 32


def kernel(layout, logits, value, act, old_lp, adv, ret, old_v, cfg):
    """pb_ppo_loss through _FusedPPOLoss -> (loss, stats[6], dloss/dlogits [M, n_act], dloss/dvalue [M]).
    'strided': the W = 0 instance on column views of one [M, n_act + 3] buffer whose other columns are NaN (never read);
    'packed': [M, W] rows (logits | value | zero pad), W = 8, 16 or 32 by n_act; the pad gradient must be exactly 0."""
    m, n_act = logits.shape
    if layout == 'strided':
        buf = torch.full((m, n_act + 3), float('nan'), device=DEV)
        buf[:, :n_act], buf[:, n_act + 1] = logits, value
        buf.requires_grad_(True)
        loss, st = clean_pufferl.fused_ppo_loss(buf[:, :n_act], buf[:, n_act + 1:n_act + 2], act, old_lp, adv, ret, old_v,
                                                cfg)
        loss.backward()
        return loss.detach(), st, buf.grad[:, :n_act], buf.grad[:, n_act + 1]
    w = packed_width(n_act)
    out = torch.zeros(m, w, device=DEV)
    out[:, :n_act], out[:, n_act] = logits, value
    out.requires_grad_(True)
    loss, st = clean_pufferl.fused_ppo_loss_packed(out, n_act, act, old_lp, adv, ret, old_v, cfg)
    loss.backward()
    assert bool((out.grad[:, n_act + 1:] == 0).all()), 'the packed instance writes whole rows, zero padding included'
    return loss.detach(), st, out.grad[:, :n_act], out.grad[:, n_act]


def reference(logits, value, act, old_lp, adv, ret, old_v, cfg, dtype=torch.float64):
    """reference_loss differentiated by autograd in `dtype` -> (loss, stats[6], dloss/dlogits, dloss/dvalue)."""
    la = logits.detach().to(dtype).clone().requires_grad_(True)
    va = value.detach().to(dtype).reshape(-1, 1).clone().requires_grad_(True)
    with torch.enable_grad():
        loss, st = reference_loss(la, va, act, old_lp.to(dtype), adv.to(dtype), ret.to(dtype), old_v.to(dtype), cfg)
        loss.backward()
    return loss.detach(), st, la.grad, va.grad[:, 0]


def rel_err(g, gr):
    """max |g - gr| / max |gr|."""
    return float((g.double() - gr.double()).abs().max()) / (float(gr.double().abs().max()) + 1e-30)


def close_to(g, gr, tol):
    """max |g - gr| within tol of max |gr|."""
    return rel_err(g, gr) <= tol


def finite(*ts):
    return all(bool(torch.isfinite(t).all()) for t in ts)


# ---------------------------------------------------------------------------------------------------------------------
# masked actions

MASKS = ['first', 'last', 'interleaved', 'all_but_taken']


def masked_rows(m, n_act, kind, gen):
    """-> (mask [m, n_act], actions): 1 to n_act - 1 masked columns; the taken action is never masked (the samplers never
    draw a zero-probability action)."""
    if kind == 'all_but_taken':
        act = torch.randint(0, n_act, (m,), device=DEV, generator=gen)
        mask = torch.ones(m, n_act, dtype=torch.bool, device=DEV)
        mask[torch.arange(m, device=DEV), act] = False
        return mask, act
    cols = {'first': [0], 'last': [n_act - 1], 'interleaved': list(range(1, n_act, 2))}[kind]
    mask = torch.zeros(m, n_act, dtype=torch.bool, device=DEV)
    mask[:, cols] = True
    allowed = (~mask[0]).nonzero()[:, 0]
    act = allowed[torch.randint(0, allowed.numel(), (m,), device=DEV, generator=gen)]
    return mask, act


def clip_offsets(m, gen):
    """u with |u| in [0, 0.9) on half the rows and in (1.1, 3] on the rest, random sign (util_update.clip_offsets with a
    generator): 1 + c u is inside or outside [1 - c, 1 + c], never within 0.1 c of an edge, so fp32 and fp64 take the
    same branch of every clamp and maximum."""
    inside = torch.rand(m, device=DEV, generator=gen) < 0.5
    u = torch.where(inside, 0.9 * torch.rand(m, device=DEV, generator=gen),
                    1.1 + 1.9 * torch.rand(m, device=DEV, generator=gen))
    return u.double() * torch.where(torch.rand(m, device=DEV, generator=gen) < 0.5, -1.0, 1.0).double()


def away_from_edges(logits, act, value, cfg, gen):
    """-> (old_lp, old_v, ret) with every row's ratio and value change at least 0.1 clip from the clamp edges, and the
    returns at least 0.05 from the tie of the two value losses (where the value gradient jumps)."""
    m = logits.shape[0]
    with torch.no_grad():
        nl = torch.log_softmax(logits.double(), 1).gather(1, act[:, None])[:, 0]
    old_lp = (nl - torch.log1p(cfg.clip_coef * clip_offsets(m, gen))).float()
    old_v = (value.double() - cfg.vf_clip_coef * clip_offsets(m, gen)).float()
    v, ov = value.double(), old_v.double()
    mid = (v + ov + torch.clamp(v - ov, -cfg.vf_clip_coef, cfg.vf_clip_coef)) / 2
    ret = mid + torch.randn(m, device=DEV, generator=gen, dtype=torch.float64)
    gap = ret - mid
    ret = torch.where(gap.abs() < 0.05, mid + torch.where(gap < 0, -0.05, 0.05), ret).float()
    return old_lp, old_v, ret


@pytest.mark.parametrize('m', MS)
@pytest.mark.parametrize('n_act', [2, 4, 7, 8, 15, 16, 31])
@pytest.mark.parametrize('layout', LAYOUTS)
def test_masked_logits_give_finite_loss_and_zero_gradient(m, n_act, layout):
    """Masked columns at -inf (masked_fill), finfo(float32).min and -1e30: the loss and the six statistics are finite and
    within test_gpu_ppo_loss.py's tolerances of fp64 (1e-5 relative, 1e-6 absolute); the masked columns' gradients are
    exactly 0, as autograd's are, and every gradient is within 1e-5 of the largest.  The entropy takes a masked logit as
    max(z - lse, -FLT_MAX) (cleanrl.entropy's clamp), and its gradient term p_j (nl_j + H) is 0 where p_j = 0.  Rows keep
    away from the branch edges (away_from_edges), which the edge tests below cover."""
    gen = torch.Generator(device=DEV).manual_seed(1000 * n_act + m)
    cfg = loss_cfg()
    for kind in MASKS:
        mask, act = masked_rows(m, n_act, kind, gen)
        base = 2.0 * torch.randn(m, n_act, device=DEV, generator=gen)
        value = torch.randn(m, device=DEV, generator=gen)
        adv = torch.randn(m, device=DEV, generator=gen)
        for fill in (float('-inf'), FMIN, -1e30):
            logits = base.masked_fill(mask, fill)
            old_lp, old_v, ret = away_from_edges(logits, act, value, cfg, gen)
            args = (logits, value, act, old_lp, adv, ret, old_v, cfg)
            loss_r, st_r, gl_r, gv_r = reference(*args)
            assert finite(loss_r, st_r, gl_r, gv_r) and bool((gl_r[mask] == 0).all())       # the reference is finite
            loss, st, gl, gv = kernel(layout, *args)
            what = (kind, fill)
            print(f'[masked] {kind} {fill:g}: gradient {rel_err(gl, gl_r):.2e}, value gradient {rel_err(gv, gv_r):.2e}, '
                  f'statistics {float((st.double() - st_r).abs().max()):.2e} (abs)', flush=True)
            assert finite(loss, st, gl, gv), what
            assert torch.allclose(loss.double(), loss_r, rtol=1e-5, atol=1e-6), (what, float(loss), float(loss_r))
            assert torch.allclose(st.double(), st_r, rtol=1e-5, atol=1e-6), (what, st, st_r)
            assert bool((gl[mask] == 0).all()), what
            assert close_to(gl, gl_r, 1e-5) and close_to(gv, gv_r, 1e-5), what


# ---------------------------------------------------------------------------------------------------------------------
# logits with a large common offset

SHIFT_ROWS = {'zeros2': [0.0, 0.0], 'half2': [0.0, -1.5], 'rand4': 4, 'rand16': 16, 'rand31': 31}


@pytest.mark.parametrize('m', MS)
@pytest.mark.parametrize('c', [0.0, 1e3, 1e5, 1e7])
@pytest.mark.parametrize('rows', list(SHIFT_ROWS))
@pytest.mark.parametrize('layout', LAYOUTS)
def test_shifted_logits_renormalise_the_entropy(m, c, rows, layout):
    """Logits + C (C = 1e3, 1e5, 1e7; fp32, so both sides see the same numbers).  lse lies on the grid of ulp(C), so
    log-probabilities carry up to ulp(C)/2 of rounding and the unnormalised p_k = exp(z_k - lse) sum to T != 1 (for
    [0, 0] + 1e5, T = 0.9978).  The logprob-derived statistics (pg, old_approx_kl, approx_kl) are within max(1e-5,
    ulp(C)) of fp64, the value loss within 1e-5; the entropy is within 1e-5 of cleanrl.entropy in fp32, which
    renormalises through its softmax (1 - 2^-20 < T < 1 + 2^-20 leaves the probabilities as they are).  Up to C = 1e5 the
    logit gradients are within max(1e-5, ulp(C)) of fp64's largest (the ratio carries the logprob's rounding; the entropy
    term does not, a shift of lse cancels in nl_j + H).  At C = 1e7 the logprob's rounding (up to 0.5) moves ratios
    across the clip edge, where the gradient changes branch, so neither the gradients nor clipfrac are compared there;
    clipfrac is left out at every C for the same reason."""
    gen = torch.Generator(device=DEV).manual_seed(m + int(c) % 9973 + len(rows))
    spec = SHIFT_ROWS[rows]
    if isinstance(spec, list):
        base = torch.tensor(spec, device=DEV).expand(m, len(spec)).contiguous()
    else:
        base = torch.randn(m, spec, device=DEV, generator=gen)
    n_act = base.shape[1]
    logits = base + c
    cfg = loss_cfg()
    act = torch.randint(0, n_act, (m,), device=DEV, generator=gen)
    with torch.no_grad():
        nl = torch.log_softmax(logits.double(), 1).gather(1, act[:, None])[:, 0]
    old_lp = (nl + 0.05 * (2 * torch.rand(m, device=DEV, generator=gen, dtype=torch.float64) - 1)).float()
    value = torch.randn(m, device=DEV, generator=gen)
    adv = 2 * torch.rand(m, device=DEV, generator=gen) - 1
    _, old_v, ret = away_from_edges(logits, act, value, cfg, gen)
    args = (logits, value, act, old_lp, adv, ret, old_v, cfg)
    _, st_r, gl_r, gv_r = reference(*args)
    loss, st, gl, gv = kernel(layout, *args)
    tol = max(1e-5, float(np.spacing(np.float32(c))))
    ent32 = float(cleanrl.entropy(logits - logits.logsumexp(-1, keepdim=True)).double().mean())
    print(f'[shifted] {rows} C={c:g}: pg/okl/kl {max(abs(float(st[k]) - float(st_r[k])) for k in (0, 3, 4)) / tol:.2f} of '
          f'tol {tol:.1e}, entropy {abs(float(st[2]) - ent32):.2e}, gradient {rel_err(gl, gl_r):.2e}', flush=True)
    assert finite(loss, st, gl, gv)
    for k, name in ((0, 'pg'), (3, 'old_approx_kl'), (4, 'approx_kl')):
        assert abs(float(st[k]) - float(st_r[k])) <= tol, (name, float(st[k]), float(st_r[k]), tol)
    assert abs(float(st[1]) - float(st_r[1])) <= 1e-5 * abs(float(st_r[1])) + 1e-6
    assert abs(float(st[2]) - ent32) <= 1e-5, (float(st[2]), ent32, float(st_r[2]))
    assert close_to(gv, gv_r, 1e-5)
    if c <= 1e5:
        assert close_to(gl, gl_r, tol), float((gl.double() - gl_r).abs().max())


# ---------------------------------------------------------------------------------------------------------------------
# exact branch edges

# value-loss rows, all with v = 1 and vclip = 0.25 (dyadic: fp32 and fp64 compute the same numbers):
#   old value 0.75 / 1.25: v - old_v = +-vclip exactly; the clipped value is v, so the two losses tie too
#   old value 0.5 / 1.5, returns 0.875 / 1.125: clipped, and the returns at the midpoint where both losses tie
VALUE_ROWS = [(0.75, 0.0), (1.25, 2.0), (0.5, 0.875), (1.5, 1.125)]
VCLIP = 0.25


def edge_rows(m, n_act, side, gen):
    """Zero logits (every row's logprob is -log(n_act), computed on the device) and v = 1; the old logprob puts the
    ratio of every third row exactly on the edge 1 + clip (side +1) or 1 - clip (side -1), with clip = |r - 1| for the
    device's own r = exp(logratio) in fp32.  The other rows lie inside (|r - 1| ~ 0.02) or outside (~0.3) the range.
    Advantages are 0 on rows 4, 9, 14, ...; value rows cycle through VALUE_ROWS.  -> (args, clip, is_edge, is_out)."""
    logits = torch.zeros(m, n_act, device=DEV)
    act = torch.randint(0, n_act, (m,), device=DEV, generator=gen)
    with torch.no_grad():
        _, nlp, _ = cleanrl.sample_logits(logits, act)          # fp32 on the device, as the kernel computes it
    i = torch.arange(m, device=DEV)
    kind = i % 3                                                # 0: on the edge, 1: inside, 2: outside
    step = torch.where(kind == 0, 0.125, torch.where(kind == 1, 0.02, 0.3)) * side
    old_lp = nlp - step
    r = (nlp - old_lp).exp()
    clip = abs(float(r[0]) - 1.0)                               # fp32 r - 1 is exact: 1 +- clip == r bit for bit
    assert bool((r[kind == 0] == r[0]).all())
    adv = torch.randn(m, device=DEV, generator=gen)
    adv[i % 5 == 4] = 0.0
    vr = torch.tensor(VALUE_ROWS, device=DEV)[i % len(VALUE_ROWS)]
    value = torch.ones(m, device=DEV)
    args = (logits, value, act, old_lp, adv, vr[:, 1], vr[:, 0], loss_cfg(clip=clip, vclip=VCLIP))
    return args, clip, kind == 0, kind == 2


@pytest.mark.parametrize('m', MS)
@pytest.mark.parametrize('side', [1, -1])
@pytest.mark.parametrize('layout,n_act', [('strided', 2), ('packed', 2), ('packed', 8), ('packed', 16)],
                         ids=['W0', 'W8', 'W16', 'W32'])
def test_ratio_and_value_edges_follow_aten(m, side, layout, n_act):
    """Rows exactly at ratio = 1 +- clip, at v - old_v = +-vclip, at the tie of the clipped and unclipped value losses, and
    with zero advantages.  ATen's rules: clamp passes the gradient at its bounds (so a ratio on the edge, where the two
    policy losses tie and maximum splits the gradient, gets all of -adv, not half), and maximum splits a tie of the value
    losses (v = 1, old value 0.5, returns 0.875: half of 2 (v - ret), the clipped half being blocked).  The logit
    gradients and the statistics are compared with autograd of the fp32 formulation on the same ratio (fp64's exp would
    move the edge rows off the edge), the value gradient and value loss with fp64 (their rows are dyadic), within 1e-6;
    clipfrac counts exactly the outside rows (the edge rows are inside: |r - 1| > clip is false).  The per-row arrays are
    strided column views, as fused_ppo_loss accepts them."""
    gen = torch.Generator(device=DEV).manual_seed(m + 7 * n_act + side)
    args, clip, edge, out = edge_rows(m, n_act, side, gen)
    _, st32, gl32, _ = reference(*args, dtype=torch.float32)
    _, st_r, _, gv_r = reference(*args)
    loss, st, gl, gv = kernel(layout, *args)
    print(f'[edges] gradient {rel_err(gl, gl32):.2e}, value gradient {rel_err(gv, gv_r):.2e}', flush=True)
    assert float(st32[5]) * m == pytest.approx(int(out.sum()))
    assert round(float(st[5]) * m) == int(out.sum()), 'the kernel must see the edge rows inside the clip range'
    assert torch.allclose(st, st32, rtol=1e-5, atol=1e-6), (st, st32)
    assert abs(float(st[1]) - float(st_r[1])) <= 1e-6 * float(st_r[1])
    assert close_to(gl, gl32, 1e-6), float((gl - gl32).abs().max())
    assert close_to(gv, gv_r, 1e-6), float((gv.double() - gv_r).abs().max())
    # the rule itself on the edge rows: d loss / d ratio = -adv (not -adv / 2), so the taken action's logit gets
    # -adv r / M (1 - 1 / n_act); the entropy term vanishes on uniform rows (nl_j + H = 0)
    act, adv = args[2], args[4]
    rows = edge & (adv != 0)
    assert bool(rows.any())
    g_a = gl[rows].gather(1, act[rows][:, None])[:, 0]
    expect = -adv[rows] * (1.0 + side * clip) / m * (1 - 1 / n_act)
    assert close_to(g_a, expect, 1e-6), float((g_a - expect).abs().max())


# ---------------------------------------------------------------------------------------------------------------------
# the k_mlp_update loss epilogue at the same edges

@pytest.mark.parametrize('m', [1, 255, 256, 257, 65537])
@pytest.mark.parametrize('side', [1, -1])
@pytest.mark.parametrize('n_act', [2, 7])
def test_mlp_update_epilogue_edges(m, side, n_act):
    """pb_mlp_update_fused with W_cat = 0: every head output is b_cat exactly (zero logits, value 1), so edge_rows'
    rows reach ppo_row_sub unchanged.  Its dOut dump (util_update.fused, debug) follows the ATen rules within 1e-6 of the
    fp32 autograd formulation (logits) and fp64 (value), and its clipfrac counts exactly the outside rows."""
    gen = torch.Generator(device=DEV).manual_seed(31 * m + n_act + side)
    args, clip, _, out = edge_rows(m, n_act, side, gen)
    logits, value, act, old_lp, adv, ret, old_v, cfg = args
    ret, old_v = ret.contiguous(), old_v.contiguous()              # the kernel reads contiguous per-row arrays
    _, _, gl32, _ = reference(*args, dtype=torch.float32)
    _, _, _, gv_r = reference(*args)
    x = torch.randn(m + 64, 128, device=DEV, generator=gen)
    w_enc = 0.1 * torch.randn(128, 128, device=DEV, generator=gen)
    b_enc = 0.1 * torch.randn(128, device=DEV, generator=gen)
    w_cat = torch.zeros(8, 128, device=DEV)
    b_cat = torch.zeros(8, device=DEV)
    b_cat[n_act] = 1.0
    fcfg = (cfg.clip_coef, 1, cfg.vf_clip_coef, cfg.vf_coef, cfg.ent_coef)
    _, stats, _, _, do, _ = uu.fused(x, 128, m, m, 1, w_enc, b_enc, w_cat, b_cat, act, old_lp, adv, ret, old_v, n_act, True,
                                     cfg=fcfg)
    torch.cuda.synchronize()
    print(f'[epilogue] gradient {rel_err(do[:, :n_act], gl32):.2e}, value gradient {rel_err(do[:, n_act], gv_r):.2e}',
          flush=True)
    assert finite(do[:, :n_act + 1], stats[:6])
    assert int(round(float(stats[5]))) == int(out.sum()), 'the kernel must see the edge rows inside the clip range'
    assert close_to(do[:, :n_act], gl32, 1e-6), float((do[:, :n_act] - gl32).abs().max())
    assert close_to(do[:, n_act], gv_r, 1e-6), float((do[:, n_act].double() - gv_r).abs().max())
    assert bool((do[:, n_act + 1:] == 0).all())


@pytest.mark.parametrize('n_act', [1, 4, 7])
def test_mlp_update_at_logit_offset(n_act):
    """util_update.case with every logit near C = 1e3 (ulp(C) = 2^-14): the stage, end-to-end and sum-of-squares checks
    hold with their usual bounds."""
    assert uu.case(4097, 1, 4097, n_act, 40 + n_act, logit_offset=1e3)


# ---------------------------------------------------------------------------------------------------------------------
# train()

class ArmsModel(torch.nn.Module):
    """A small custom policy: Linear -> ReLU -> logits / value heads; the `masked` arms are unavailable, their logits
    -inf (masked_fill), as action masks are usually applied."""

    def __init__(self, env, n_act, masked=(), hidden=32):
        super().__init__()
        n_obs = int(np.prod(env.single_observation_space.shape))
        self.enc = torch.nn.Linear(n_obs, hidden)
        self.actor = torch.nn.Linear(hidden, n_act)
        self.critic = torch.nn.Linear(hidden, 1)
        mask = torch.zeros(n_act, dtype=torch.bool)
        mask[list(masked)] = True
        self.register_buffer('mask', mask)

    def forward(self, x):
        h = torch.relu(self.enc(x.reshape(x.shape[0], -1).float()))
        return self.actor(h).masked_fill(self.mask, float('-inf')), self.critic(h)


def arms_train(monkeypatch, arms, masked, fused_sample):
    """evaluate() + train() on the bandit with an ArmsModel, fused_loss True and False from the same seed -> per run
    (rollout arrays, parameters, losses, update plan)."""
    n, h = 256, 32
    plans = []
    plan_fn = clean_pufferl.update_plan
    monkeypatch.setattr(clean_pufferl, 'update_plan', lambda d: plans.append(plan_fn(d)) or plans[-1])
    res = {}
    for fused in (True, False):
        vec = pvec.make(ocean.env_creator('bandit'), env_kwargs=dict(num_actions=arms), num_envs=n, backend=pvec.B200)
        torch.manual_seed(0)
        pol = cleanrl.Policy(ArmsModel(vec, arms, masked), fused_sample=fused_sample, seed=3).cuda()
        data = clean_pufferl.create(make_config(n, h, env='bandit', fused_loss=fused), vec, pol)
        clean_pufferl.evaluate(data)
        exp = data.experience
        roll = {k: getattr(exp, k).cpu().numpy().copy() for k in ('obs', 'actions', 'logprobs', 'values', 'rewards', 'dones')}
        clean_pufferl.train(data)
        losses = np.array([data.losses.policy_loss, data.losses.value_loss, data.losses.entropy, data.losses.approx_kl,
                           data.losses.clipfrac, data.losses.explained_variance])
        res[fused] = (roll, [p.detach().clone() for p in pol.parameters()], losses, plans[-1])
        clean_pufferl.close(data)
    return res


def assert_same_training(res):
    """The tolerances of test_pong_fused_loss_train_matches_reference_loss: the same rollout, parameters within 2e-5,
    losses within 1e-4 relative."""
    for k in res[True][0]:
        assert np.array_equal(res[True][0][k], res[False][0][k]), k
    for p in res[True][1]:
        assert finite(p)
    d = torch.cat([(a - b).abs().flatten() for a, b in zip(res[True][1], res[False][1])])
    lt, lf = res[True][2], res[False][2]
    print(f'parameters: max diff {float(d.max()):.2e}; losses fused {lt} reference {lf}', flush=True)
    assert np.isfinite(lt).all()
    assert float(d.max()) <= 2e-5
    assert np.allclose(lt, lf, rtol=1e-4, atol=1e-6), (lt, lf)


def test_masked_policy_train_matches_reference_loss(monkeypatch):
    """A 6-arm bandit whose arms 1 and 4 are unavailable (-inf logits): the rollout never draws them, and train() on the
    'model' engine (the policy's forward, pb_ppo_loss, autograd) matches fused_loss=False (the reference loss)."""
    res = arms_train(monkeypatch, 6, (1, 4), fused_sample=True)
    assert (res[True][3].engine, res[False][3].engine) == ('model', 'reference')
    acts = res[True][0]['actions']
    assert not np.isin(acts, [1, 4]).any() and np.isin(acts, [0, 2, 3, 5]).all()
    assert_same_training(res)


def test_more_than_32_actions_train_on_the_reference_loss(monkeypatch):
    """A 40-action head is past pb_ppo_loss's 32: update_plan sends it to the reference loss, and train() matches
    fused_loss=False (it raised in pb_ppo_loss before)."""
    res = arms_train(monkeypatch, 40, (3, 17, 39), fused_sample=False)
    assert res[True][3].engine == 'reference' and res[False][3].engine == 'reference'
    assert_same_training(res)
