"""2-rank hardware check of the NVLink peer-memory all-reduce and the one-graph multi-GPU update (torchrun):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 \
        tests/multi_gpu/check_peer_update.py

1. PeerComm.all_reduce_ against torch.distributed.all_reduce (NCCL) on random buffers, 200 back-to-back calls, eager and
   inside a CUDA graph (bit-identical results on both ranks).
2. breakout through create/evaluate/train on every rank (env shards by global index): the hand-written update with the
   fused peer all-reduce must leave bit-identical parameters on all ranks, match the NCCL fallback path to fp32 noise,
   and run as ONE captured graph (train_graph_state == 2).
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


def check_allreduce(rank, world):
    comm = pdist.PeerComm(20000)
    torch.manual_seed(100 + rank)
    for n in (1, 17157, 20000):
        x = torch.randn(n, device='cuda')
        ref = x.clone()
        dist.all_reduce(ref)
        got = comm.all_reduce_(x.clone())
        torch.cuda.synchronize()
        err = float((got - ref).abs().max())
        assert err <= 1e-5 * max(1.0, float(ref.abs().max())), (n, err)
        other = [torch.empty_like(got) for _ in range(world)]
        dist.all_gather(other, got)
        assert all(torch.equal(o, got) for o in other), 'ranks must hold bit-identical sums'
    # many back-to-back calls (epoch protocol, slot reuse), then the same inside a CUDA graph
    x = torch.randn(17157, device='cuda')
    acc = x.clone()
    for _ in range(200):
        comm.all_reduce_(acc)
        acc.mul_(1.0 / world)
    torch.cuda.synchronize()
    ref = x.clone()
    for _ in range(3):
        dist.all_reduce(ref)
        ref.mul_(1.0 / world)
    buf = x.clone()
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        for _ in range(3):
            comm.all_reduce_(buf)
            buf.mul_(1.0 / world)
    buf.copy_(x)
    g.replay()
    torch.cuda.synchronize()
    assert float((buf - ref).abs().max()) <= 1e-5, float((buf - ref).abs().max())
    # timing: 16 calls per replay, like one PPO step
    buf2 = torch.randn(17157, device='cuda')
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        for _ in range(16):
            comm.all_reduce_(buf2)
    g2.replay()
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        g2.replay()
    e1.record()
    torch.cuda.synchronize()
    log(rank, f'peer all-reduce of 68.6 KB: {e0.elapsed_time(e1) * 1000 / 160:.2f} us per call (graph replay, {world} ranks)')
    e0.record()
    for _ in range(160):
        dist.all_reduce(buf2)
    e1.record()
    torch.cuda.synchronize()
    log(rank, f'NCCL all_reduce of 68.6 KB:  {e0.elapsed_time(e1) * 1000 / 160:.2f} us per call (eager)')
    comm.close()


def run_train(rank, world, peer, iters=2, n=2048, h=128):
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=n,
                    backend=pvec.B200.options(exact_infos=False, env_index_offset=rank * n))
    torch.manual_seed(1)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=1 + rank).cuda()
    pdist.broadcast_parameters(pol)
    cfg = pufferlib_b200.namespace(
        seed=1, torch_deterministic=True, env='breakout', batch_size=n * h, bptt_horizon=16, minibatch_size=n * h // 4,
        cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
        update_epochs=2, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5, ent_coef=0.01,
        max_grad_norm=0.5, target_kl=None, anneal_lr=False, total_timesteps=10 ** 10, cuda_graph=True,
        peer_allreduce=peer)
    data = clean_pufferl.create(cfg, vec, pol)
    for _ in range(iters):
        clean_pufferl.evaluate(data)
        clean_pufferl.train(data)
    torch.cuda.synchronize()
    flat = torch.cat([p.detach().reshape(-1) for p in pol.parameters()])
    state = (data.train_graph_state, data.manual_update is not None, data.manual_update.peer is not None if data.manual_update else None)
    clean_pufferl.close(data)
    return flat, state, data


def main():
    rank, local, world = pdist.init()
    torch.cuda.set_device(local)
    check_allreduce(rank, world)
    log(rank, 'peer all-reduce: ok')
    flat_peer, st_peer, _ = run_train(rank, world, peer=True)
    others = [torch.empty_like(flat_peer) for _ in range(world)]
    dist.all_gather(others, flat_peer)
    assert all(torch.equal(o, flat_peer) for o in others), 'parameters diverged between ranks'
    assert st_peer == (2, True, True), st_peer
    log(rank, f'one-graph update with fused peer all-reduce: ok (state {st_peer})')
    flat_nccl, st_nccl, _ = run_train(rank, world, peer=False)
    assert st_nccl[1] and st_nccl[2] is False, st_nccl
    # same rollouts (deterministic envs + per-rank sampler seeds), same math, different summation order of the rank sums
    diff = float((flat_peer - flat_nccl).abs().max())
    log(rank, f'peer vs NCCL-fallback parameters after 2 iterations: max abs diff {diff:.3e}')
    assert diff < 5e-4, diff
    log(rank, 'ALL OK')
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
