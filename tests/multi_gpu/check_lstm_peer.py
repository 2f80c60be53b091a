"""2-rank hardware check of the recurrent update on several GPUs (torchrun, one node):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29513 \
        tests/multi_gpu/check_lstm_peer.py

RecurrentPolicy(LSTMWrapper(Default), fused_sample=True, fused_update=True) trains breakout, every rank on its own env
shard, so the ranks' gradients and approx_kl differ.  A probe call (target_kl = 1e9, peer exchange) reads each rank's
approx_kl of epoch 0's last minibatch; target_kl is then set between the smallest and the largest, so a rank deciding on its
own would stop after another epoch than its peer.  Two plans run three evaluate + train() calls each: the gradient mean
over NVLink peer memory (pb_peer_allreduce_mean), whose update must be captured whole (train_graph_state == 2), and the
same without peers (NCCL, peer_allreduce=False), which stays eager.  Every call must run the same epochs on every rank and
leave bit-identical parameters on every rank.
"""
import os
import sys

import torch
import torch.distributed as dist

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)

import pufferlib_b200  # noqa: E402
import pufferlib_b200.vector as pvec  # noqa: E402
from pufferlib_b200 import clean_pufferl, models, distributed as pdist  # noqa: E402
from pufferlib_b200.environments import ocean  # noqa: E402
from pufferlib_b200.frameworks import cleanrl  # noqa: E402


def log(rank, *a):
    if rank == 0:
        print(*a, flush=True)


def make(rank, target_kl, n=1024, h=64, **kw):
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=n,
                    backend=pvec.B200.options(exact_infos=False, env_index_offset=rank * n))
    torch.manual_seed(1)
    net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env), input_size=128, hidden_size=128)
    pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=1 + rank, fused_update=True).cuda()
    pdist.broadcast_parameters(pol)
    cfg = pufferlib_b200.namespace(
        seed=1, torch_deterministic=True, env='breakout', batch_size=n * h, bptt_horizon=16, minibatch_size=n * h // 4,
        cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
        update_epochs=4, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01,
        max_grad_norm=0.5, target_kl=target_kl, anneal_lr=False, total_timesteps=10 ** 10, cuda_graph=True, **kw)
    return clean_pufferl.create(cfg, vec, pol), pol


def gathered(x):
    out = [torch.empty_like(x) for _ in range(dist.get_world_size())]
    dist.all_gather(out, x)
    return out


def probe_target(rank):
    """A target_kl between the ranks' own approx_kl of epoch 0's last minibatch (the KL row sum the exchange carries)."""
    data, _ = make(rank, 1e9)
    seen = []
    real = pdist.GradBucket.peer_all_reduce_mean

    def record(self, kl_in=None, kl_out=None):
        if kl_in is not None:
            seen.append(kl_in.clone())
        return real(self, kl_in, kl_out)
    pdist.GradBucket.peer_all_reduce_mean = record
    try:
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)           # eager: the first call
    finally:
        pdist.GradBucket.peer_all_reduce_mean = real
    assert data.grad_bucket.peer is not None, data.msg
    own = (seen[0].float() / data.experience.minibatch_size).reshape(1)
    kls = [float(k) for k in gathered(own)]
    clean_pufferl.close(data)
    assert max(kls) > min(kls), kls
    return (min(kls) * max(kls)) ** 0.5, kls


def run_plan(rank, name, target, **kw):
    data, pol = make(rank, target, **kw)
    epochs = []
    for _ in range(3):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
        torch.cuda.synchronize()
        ran = [int(e) for e in gathered(torch.tensor([data.train_epochs_run], device='cuda'))]
        assert len(set(ran)) == 1, f'{name}: ranks ran different epochs {ran}'
        epochs.append(ran[0])
        flat = torch.cat([p.detach().reshape(-1) for p in pol.parameters()])
        assert all(torch.equal(o, flat) for o in gathered(flat)), f'{name}: parameters diverged between ranks'
    state = (data.train_graph_state, data.train_recurrent_path, data.grad_bucket.peer is not None)
    clean_pufferl.close(data)
    log(rank, f'{name}: epochs run {epochs} on every rank, parameters bit-identical, state {state}')
    return state


def main():
    rank, local, world = pdist.init()
    torch.cuda.set_device(local)
    target, kls = probe_target(rank)
    log(rank, f'own approx_kl of epoch 0 per rank {kls}; target_kl {target:.6g}')
    st = run_plan(rank, 'peer, captured', target)
    assert st == (2, 'fused', True), st
    st = run_plan(rank, 'NCCL fallback', target, peer_allreduce=False)
    assert st[1] == 'fused' and not st[2] and st[0] != 2, st
    log(rank, 'ALL OK')
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
