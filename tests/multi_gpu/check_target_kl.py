"""2-rank hardware check of target_kl on several GPUs (torchrun, one node):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29512 \
        tests/multi_gpu/check_target_kl.py

Every rank trains breakout on its own env shard, so the ranks' approx_kl differ.  A probe call (target_kl = 1e9) reads
each rank's approx_kl of epoch 0's last minibatch; target_kl is then set between the smallest and the largest, so a rank
deciding on its own would stop after another epoch than its peer.  Three plans run three evaluate + train() calls each:
the hand-written update with the peer exchange, captured (train_graph_state == 2), the same without peers (NCCL,
peer_allreduce=False) and autograd (manual_update=False).  Every call must run the same epochs on every rank and leave
bit-identical parameters on every rank; a rank stopping alone would leave its peer's next all-reduce without a partner.
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


def make(rank, target_kl, n=2048, h=128, **kw):
    vec = pvec.make(ocean.env_creator('breakout'), num_envs=n,
                    backend=pvec.B200.options(exact_infos=False, env_index_offset=rank * n))
    torch.manual_seed(1)
    pol = cleanrl.Policy(models.Default(vec.driver_env), fused_sample=True, seed=1 + rank).cuda()
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
    """A target_kl between the ranks' own approx_kl of epoch 0's last minibatch."""
    data, _ = make(rank, 1e9)
    clean_pufferl.evaluate(data)
    clean_pufferl.train(data)
    mu = data.manual_update
    nm = data.experience.num_minibatches
    own = (mu.stats[nm - 1, 4] / mu.mb_rows).reshape(1)
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
    state = (data.train_graph_state, data.manual_update is not None,
             data.manual_update is not None and data.manual_update.peer is not None)
    clean_pufferl.close(data)
    log(rank, f'{name}: epochs run {epochs} on every rank, parameters bit-identical, state {state}')
    return state


def main():
    rank, local, world = pdist.init()
    torch.cuda.set_device(local)
    target, kls = probe_target(rank)
    log(rank, f'own approx_kl of epoch 0 per rank {kls}; target_kl {target:.6g}')
    st = run_plan(rank, 'peer, captured', target)
    assert st == (2, True, True), st
    st = run_plan(rank, 'NCCL fallback', target, peer_allreduce=False)
    assert st[1] and not st[2], st
    st = run_plan(rank, 'autograd', target, manual_update=False)
    assert not st[1], st
    log(rank, 'ALL OK')
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
