"""A small instance of the fused recurrent policy step (pb_policy_lstm_sample, csrc/policy_lstm.cu) for compute-sanitizer
(memcheck / racecheck / synccheck), next to sanitize_targets.py:

    compute-sanitizer --tool memcheck python tests/experimental/sanitize_lstm.py

200 envs leave the last CTA partially filled (rows >= m must be neither read nor written); one rollout of 16 steps through
clean_pufferl.evaluate (in-place lstm_h / lstm_c update, rollout rows written by the kernel) and one update."""
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
import pufferlib_b200  # noqa: E402
import pufferlib_b200.vector as pvec  # noqa: E402
from pufferlib_b200 import clean_pufferl, models  # noqa: E402
from pufferlib_b200.environments import ocean  # noqa: E402
from pufferlib_b200.frameworks import cleanrl  # noqa: E402

n, h = 200, 16
cfg = pufferlib_b200.namespace(
    seed=1, torch_deterministic=True, env='squared', batch_size=n * h, bptt_horizon=16, minibatch_size=n * h // 2,
    cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95, update_epochs=1,
    norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01, max_grad_norm=0.5,
    target_kl=None, anneal_lr=False, total_timesteps=10 ** 9)
vec = pvec.make(ocean.env_creator('squared'), num_envs=n, backend=pvec.B200)
torch.manual_seed(0)
net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1).cuda()
data = clean_pufferl.create(cfg, vec, pol)
clean_pufferl.evaluate(data)
clean_pufferl.train(data)
torch.cuda.synchronize()
assert np.isfinite(data.losses.policy_loss) and int(pol._counter[0]) == h
clean_pufferl.close(data)
print('lstm ok', flush=True)
