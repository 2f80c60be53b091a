"""A small instance of each ocean test env kind (csrc/env_ocean.cu) for compute-sanitizer, next to sanitize_lstm.py:

    compute-sanitizer --tool memcheck python tests/experimental/sanitize_ocean.py

37 envs leave the last warp of every step kernel partially filled; memory's reset-sends run k_mem_prepare over a
twist boundary (37 * 13 outputs per reset-send at mem_length=5, mem_delay=3); password runs 100 floats per obs row;
bandit builds its gaussian table.  Each kind: reset, then sends with random actions, with exact infos."""
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
import pufferlib_b200.vector as pvec  # noqa: E402
from pufferlib_b200.environments import ocean  # noqa: E402

n = 37
rng = np.random.default_rng(0)
for kind, kw in (('memory', {'mem_length': 5, 'mem_delay': 3}), ('password', {'password_length': 100}),
                 ('stochastic', {}), ('bandit', {'num_actions': 33})):
    vec = pvec.make(ocean.env_creator(kind), env_kwargs=kw, num_envs=n, backend=pvec.B200.options(exact_infos=True))
    vec.async_reset(3)
    for _ in range(40):
        vec.recv()
        vec.send(rng.integers(0, vec.single_action_space.n, size=n))
    vec.recv()
    torch.cuda.synchronize()
    vec.close()
print('ocean envs ok', flush=True)
