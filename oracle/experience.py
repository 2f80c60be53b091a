"""``clean_pufferl.Experience`` + the train-side prep, restated in numpy.  TEST INFRASTRUCTURE.

Follows reference clean_pufferl.py:
  :382-434  __init__  (flat [batch_size] arrays in arrival (ptr) order, validation errors)
  :436-450  store     (masked rows appended at ptr; sort key (env_id, step) per row)
  :452-464  sort_training_data  (lexicographic argsort -> idxs; b_idxs_obs = idxs.reshape(rows, n_mb, bptt).transpose(1,0,2))
  :466-482  flatten_batch       (b_advantages regroup; returns_np = advantages_np + values_np [sic: sorted + arrival order])
  :211-213  per-minibatch advantage normalisation, Bessel-corrected std, +1e-8 on the std
"""
import numpy as np


class Experience:
    def __init__(self, batch_size, bptt_horizon, minibatch_size, obs_shape, obs_dtype, atn_shape=()):
        if minibatch_size is None:
            minibatch_size = batch_size
        self.obs = np.zeros((batch_size, *obs_shape), dtype=obs_dtype)
        self.actions = np.zeros((batch_size, *atn_shape), dtype=np.int64)
        self.logprobs = np.zeros(batch_size, dtype=np.float32)
        self.rewards = np.zeros(batch_size, dtype=np.float32)
        self.dones = np.zeros(batch_size, dtype=np.float32)
        self.truncateds = np.zeros(batch_size, dtype=np.float32)   # never written (reference quirk)
        self.values = np.zeros(batch_size, dtype=np.float32)
        num_minibatches = batch_size / minibatch_size
        self.num_minibatches = int(num_minibatches)
        if self.num_minibatches != num_minibatches:
            raise ValueError('batch_size must be divisible by minibatch_size')
        minibatch_rows = minibatch_size / bptt_horizon
        self.minibatch_rows = int(minibatch_rows)
        if self.minibatch_rows != minibatch_rows:
            raise ValueError('minibatch_size must be divisible by bptt_horizon')
        self.batch_size = batch_size
        self.bptt_horizon = bptt_horizon
        self.minibatch_size = minibatch_size
        self.sort_keys = []
        self.ptr = 0
        self.step = 0

    @property
    def full(self):
        return self.ptr >= self.batch_size

    def store(self, obs, value, action, logprob, reward, done, env_id, mask):
        ptr = self.ptr
        indices = np.where(np.asarray(mask))[0][:self.batch_size - ptr]
        end = ptr + len(indices)
        self.obs[ptr:end] = np.asarray(obs)[indices]
        self.values[ptr:end] = np.asarray(value)[indices]
        self.actions[ptr:end] = np.asarray(action)[indices]
        self.logprobs[ptr:end] = np.asarray(logprob)[indices]
        self.rewards[ptr:end] = np.asarray(reward)[indices]
        self.dones[ptr:end] = np.asarray(done)[indices]
        self.sort_keys.extend([(int(env_id[i]), self.step) for i in indices])
        self.ptr = end
        self.step += 1

    def sort_training_data(self):
        idxs = np.asarray(sorted(range(len(self.sort_keys)), key=self.sort_keys.__getitem__))
        self.b_idxs_obs = idxs.reshape(self.minibatch_rows, self.num_minibatches,
                                       self.bptt_horizon).transpose(1, 0, 2)
        self.b_idxs = self.b_idxs_obs
        self.b_idxs_flat = self.b_idxs.reshape(self.num_minibatches, self.minibatch_size)
        self.sort_keys = []
        self.ptr = 0
        self.step = 0
        return idxs

    def flatten_batch(self, advantages):
        b_idxs, b_flat = self.b_idxs, self.b_idxs_flat
        self.b_advantages = advantages.reshape(self.minibatch_rows, self.num_minibatches, self.bptt_horizon
                                               ).transpose(1, 0, 2).reshape(self.num_minibatches,
                                                                            self.minibatch_size)
        self.returns_np = advantages + self.values
        self.b_obs = self.obs[self.b_idxs_obs]
        self.b_actions = self.actions[b_idxs]
        self.b_logprobs = self.logprobs[b_idxs]
        self.b_dones = self.dones[b_idxs]
        self.b_values = self.values[b_flat]
        self.b_returns = self.b_advantages + self.b_values


def normalize_advantages(adv):
    """clean_pufferl.py:211-213 for one minibatch (fp32, unbiased std).  Reduction in float64, cast at the
    end: the fp32 torch result differs from this by summation-order rounding only (tolerance tests)."""
    a = np.asarray(adv, dtype=np.float32).reshape(-1)
    mean = np.float32(a.astype(np.float64).mean())
    std = np.float32(np.sqrt(((a.astype(np.float64) - a.astype(np.float64).mean()) ** 2).sum() / (a.size - 1)))
    return (a - mean) / (std + np.float32(1e-8))
