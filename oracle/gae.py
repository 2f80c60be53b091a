"""``c_gae.compute_gae`` restated.  TEST INFRASTRUCTURE (see oracle/__init__.py).

``compute_gae_np``  sequential numpy-fp32 loop following reference c_gae.pyx:24-30 (small cases).
``compute_gae``     ctypes call into ``oracle/csrc/gae.c`` (same recurrence in C, any size).
``compute_gae_f64`` the recurrence in float64 (C): ground truth used to put both the reference's and the
                    CUDA scan's rounding error on one scale in the tolerance tests.
"""
import ctypes
import numpy as np

from . import build as _build


def compute_gae_np(dones, values, rewards, gamma, gae_lambda):
    dones, values, rewards = (np.ascontiguousarray(a, dtype=np.float32) for a in (dones, values, rewards))
    gamma, gae_lambda = np.float32(gamma), np.float32(gae_lambda)
    n = len(rewards)
    adv = np.zeros(n, dtype=np.float32)
    last = np.float32(0)
    one = np.float32(1)
    for t in range(n - 1):
        t_cur, t_next = n - 2 - t, n - 1 - t
        nnt = one - dones[t_next]
        delta = rewards[t_next] + gamma * values[t_next] * nnt - values[t_cur]
        last = delta + gamma * gae_lambda * nnt * last
        adv[t_cur] = last
    return adv


def compute_gae(dones, values, rewards, gamma, gae_lambda):
    lib = _build.load()
    dones, values, rewards = (np.ascontiguousarray(a, dtype=np.float32) for a in (dones, values, rewards))
    n = len(rewards)
    adv = np.zeros(n, dtype=np.float32)
    fp = ctypes.POINTER(ctypes.c_float)
    lib.oracle_compute_gae(dones.ctypes.data_as(fp), values.ctypes.data_as(fp), rewards.ctypes.data_as(fp),
                           ctypes.c_float(gamma), ctypes.c_float(gae_lambda), adv.ctypes.data_as(fp),
                           ctypes.c_long(n))
    return adv


def compute_gae_f64(dones, values, rewards, gamma, gae_lambda):
    lib = _build.load()
    dones, values, rewards = (np.ascontiguousarray(a, dtype=np.float32) for a in (dones, values, rewards))
    n = len(rewards)
    adv = np.zeros(n, dtype=np.float64)
    fp = ctypes.POINTER(ctypes.c_float)
    lib.oracle_compute_gae_f64(dones.ctypes.data_as(fp), values.ctypes.data_as(fp), rewards.ctypes.data_as(fp),
                               ctypes.c_float(gamma), ctypes.c_float(gae_lambda),
                               adv.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), ctypes.c_long(n))
    return adv
