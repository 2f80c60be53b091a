"""pufferlib_b200 -- H100-native (sm_90a) env-step + PPO-rollout hot path behind PufferLib's own interfaces.

    import pufferlib_b200.vector, pufferlib_b200.clean_pufferl
    vecenv = pufferlib_b200.vector.make(pufferlib_b200.environments.ocean.env_creator('squared'),
                                        num_envs=64, backend=pufferlib_b200.vector.B200)

There is no CPU fallback: every compute call goes through libpuffer_b200.so (include/pufferlib_b200.h) and
fails loudly if the library or a CUDA device is missing.
"""
__version__ = '0.1.0'

from pufferlib_b200.namespace import namespace, Namespace  # noqa: F401
from pufferlib_b200.exceptions import APIUsageError  # noqa: F401
