"""The multiagent env kind on the GPU: the step-send and reset-send times of its env kernel and the learning budget.

    python tests/experimental/measure_multiagent.py [--num-envs 16384] [--sends 400] [--seeds 1 2 3]

Send times: vector.B200 over num_envs envs (2 * num_envs agent rows), actions on the device, outputs into the vecenv's own
buffers.  Sends alternate between step-sends and reset-sends (every step ends both agents' episodes); CUDA events around
each send() give the device time from its first enqueued operation to its last, the medians are reported per send kind.
Learning: tests/test_gpu_multiagent.run_learning per seed (models.Default, cuda_graph=True), the first iteration at which
both agents' score reached 0.9.  Prints one JSON line; writes nothing."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [REPO, os.path.join(REPO, 'tests')]
import pufferlib_b200.vector as pvec  # noqa: E402
from pufferlib_b200.environments import ocean  # noqa: E402


def send_times(n, sends, warmup=20):
    vec = pvec.make(ocean.env_creator('multiagent'), num_envs=n, backend=pvec.B200)
    a = torch.randint(0, 2, (2 * n,), dtype=torch.int64, device='cuda')
    vec.async_reset(0)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(sends)]
    for _ in range(warmup):
        vec.recv()
        vec.send(a)
    assert warmup % 2 == 0      # the first timed send is a step-send
    for i in range(sends):
        vec.recv()
        ev[i][0].record()
        vec.send(a)
        ev[i][1].record()
    torch.cuda.synchronize()
    ms = np.asarray([s.elapsed_time(e) for s, e in ev])
    vec.close()
    return float(np.median(ms[0::2]) * 1e3), float(np.median(ms[1::2]) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num-envs', type=int, default=16384)
    ap.add_argument('--sends', type=int, default=400)
    ap.add_argument('--seeds', type=int, nargs='*', default=[1, 2, 3])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    step_us, reset_us = send_times(args.num_envs, args.sends)
    out = dict(gpu=gpu, num_envs=args.num_envs, agent_rows=2 * args.num_envs, step_send_us=round(step_us, 2),
               reset_send_us=round(reset_us, 2))
    if args.seeds:
        from test_gpu_multiagent import run_learning
        out['learning_first_iteration'] = {s: run_learning(s, 60)[0] for s in args.seeds}
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
