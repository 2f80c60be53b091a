"""A small instance of the fused recurrent update (pb_lstm_bptt_forward / pb_lstm_bptt_backward, csrc/lstm_bptt.cu) for
compute-sanitizer, next to sanitize_lstm.py:

    compute-sanitizer --tool memcheck python tests/experimental/sanitize_lstm_bptt.py
    compute-sanitizer --tool racecheck python tests/experimental/sanitize_lstm_bptt.py

200 envs with bptt 8 give minibatches of 100 segments, so the last CTA of both kernels is partially filled (segments
>= B must be neither read nor written); n_act = 8 (squared) runs the 16-column head variant.  One rollout and one
train() through RecurrentPolicy(fused_update=True), then both kernels once more directly with an initial state."""
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
    seed=1, torch_deterministic=True, env='squared', batch_size=n * h, bptt_horizon=8, minibatch_size=n * h // 4,
    cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95, update_epochs=1,
    norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01, max_grad_norm=0.5,
    target_kl=None, anneal_lr=False, total_timesteps=10 ** 9)
vec = pvec.make(ocean.env_creator('squared'), num_envs=n, backend=pvec.B200)
torch.manual_seed(0)
net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1, fused_update=True).cuda()
data = clean_pufferl.create(cfg, vec, pol)
clean_pufferl.evaluate(data)
clean_pufferl.train(data)
torch.cuda.synchronize()
assert data.train_recurrent_path == 'fused' and np.isfinite(data.losses.policy_loss)

x = data.experience.b_obs[0]
state = (torch.randn(1, x.shape[0], 128, device='cuda'), torch.randn(1, x.shape[0], 128, device='cuda'))
out, n_act, _ = net.forward_packed_seq(x, state)
out.backward(torch.randn_like(out))
torch.cuda.synchronize()
assert all(bool(p.grad.isfinite().all()) for p in net.parameters())
clean_pufferl.close(data)
print('lstm bptt ok', flush=True)
