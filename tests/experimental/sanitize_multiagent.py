"""A small instance of the multiagent env kind (csrc/env_ocean.cu, two agent rows per env) for compute-sanitizer, next
to sanitize_ocean.py:

    compute-sanitizer --tool memcheck python tests/experimental/sanitize_multiagent.py

37 envs (74 agent rows) leave the last warp of the step kernel partially filled.  Reset, then sends with random actions
(alternating step- and reset-sends) into the vecenv's own buffers with exact infos, then into a bound rollout, and the
per-agent statistics read."""
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
import pufferlib_b200.vector as pvec  # noqa: E402
from pufferlib_b200 import clean_pufferl  # noqa: E402
from pufferlib_b200.environments import ocean  # noqa: E402

n = 37
rng = np.random.default_rng(0)
vec = pvec.make(ocean.env_creator('multiagent'), num_envs=n, backend=pvec.B200.options(exact_infos=True))
vec.async_reset(3)
for _ in range(40):
    vec.recv()
    vec.send(rng.integers(0, 2, size=2 * n))
vec.recv()
exp = clean_pufferl.Experience(2 * n * 8, 4, 2 * n * 8, (1,), np.float32, ())
vec.bind_rollout(exp)
for _ in range(20):
    vec.send(torch.as_tensor(rng.integers(0, 2, size=2 * n), device='cuda'))
    vec.recv()
vec.episode_stats()
torch.cuda.synchronize()
vec.close()
print('multiagent env ok', flush=True)
