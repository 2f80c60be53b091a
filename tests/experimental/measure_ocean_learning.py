"""Iterations to threshold of tests/test_gpu_ocean_learning.py's cases on several seeds (sets their budgets).

    python tests/experimental/measure_ocean_learning.py [--seeds 1 2 3] [--iters 200]

Prints one JSON line per (case, seed) and the worst seed per case, with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from test_gpu_ocean_learning import run_case   # noqa: E402


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seeds', type=int, nargs='+', default=[1, 2, 3])
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--cases', nargs='+', default=['memory_lstm', 'password', 'stochastic', 'bandit', 'memory_mlp'])
    a = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    worst = {}
    for case in a.cases:
        for seed in a.seeds:
            t0 = time.time()
            stop = case != 'memory_mlp'
            first, hist, rec = run_case(case, seed, 120 if case == 'stochastic' else (a.iters if stop else 60), stop_early=stop)
            row = dict(case=case, seed=seed, first=first, stochastic_mean_last_20=(
                           round(float(np.mean(hist[-20:])), 4) if case == 'stochastic' else None), seconds=round(time.time() - t0, 1), record=rec,
                       last=[None if m is None else round(m, 3) for m in hist[-12:]])
            print(json.dumps(row), flush=True)
            worst[case] = max(worst.get(case, -1), first if first is not None else 10 ** 9)
    print(json.dumps({'worst_first_iteration': worst}), flush=True)


if __name__ == '__main__':
    main()
