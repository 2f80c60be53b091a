"""Small instances of the hand-written kernels for compute-sanitizer (memcheck / racecheck / synccheck):

    compute-sanitizer --tool memcheck python tests/experimental/sanitize_targets.py

Sizes are tiny on purpose (the tools slow kernels down 10-100x); every kernel family of the hot path is launched at least
once: env steps, GAE (single-pass tile kernel and the general one), train-prep, PPO loss, policy step, tail backward,
clip+Adam, the fused wgmma update and the persistent rollout."""
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
import pufferlib_b200  # noqa: E402
import pufferlib_b200.vector as pvec  # noqa: E402
from pufferlib_b200 import clean_pufferl, models  # noqa: E402
from pufferlib_b200.environments import ocean  # noqa: E402
from pufferlib_b200.frameworks import cleanrl  # noqa: E402
from util_gpu import gae_device  # noqa: E402

which = sys.argv[1:] or ['gae', 'loop', 'fused']


def cfg(env, n, h, **kw):
    d = dict(seed=1, torch_deterministic=True, env=env, batch_size=n * h, bptt_horizon=16, minibatch_size=n * h // 2,
             cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
             update_epochs=1, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01,
             max_grad_norm=0.5, target_kl=None, anneal_lr=False, total_timesteps=10 ** 9)
    d.update(kw)
    return pufferlib_b200.namespace(**d)


if 'gae' in which:
    rng = np.random.default_rng(0)
    for h, n in ((128, 64), (256, 32), (17, 33), (5, 1)):          # k_gae_fast x2, k_gae x2
        r, v = rng.standard_normal((h, n)).astype(np.float32), rng.standard_normal((h, n)).astype(np.float32)
        d = (rng.random((h, n)) < 0.05).astype(np.float32)
        gae_device(r, v, d, 0.99, 0.95)
    print('gae ok', flush=True)

for name, fused in (('loop', False), ('fused', True)):
    if name not in which:
        continue
    n, h = 128, 32
    vec = pvec.make(ocean.env_creator('breakout'), env_kwargs={'max_ticks': 20}, num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=1).cuda()
    data = clean_pufferl.create(cfg('breakout', n, h, fused_rollout=fused, fused_update=fused), vec, pol)
    for _ in range(2):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
    torch.cuda.synchronize()
    assert np.isfinite(data.losses.policy_loss)
    clean_pufferl.close(data)
    print(name, 'ok', flush=True)

if 'envs' in which:
    for kind, n in (('squared', 16), ('snake', 64), ('pong', 4)):
        vec = pvec.make(ocean.env_creator(kind), num_envs=n, backend=pvec.B200)
        vec.async_reset(1)
        for _ in range(6):
            vec.recv()
            vec.send(torch.zeros(n, dtype=torch.int64, device='cuda'))
        torch.cuda.synchronize()
        vec.close()
    print('envs ok', flush=True)
