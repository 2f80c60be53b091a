"""Multi-GPU for the rollout path: env shards per rank, ONE gradient all-reduce per optimizer step.

The reference has no distributed code (SURVEY §2, §8e).  Envs are independent, so rank g owns envs
[g*N/G, (g+1)*N/G) seeded by GLOBAL env index (``env_index_offset``); rollout, GAE, advantage normalisation and
minibatching are rank-local (identical to running the reference per shard); the policy is replicated and its
gradients are averaged with a single NCCL all-reduce over one flat fp32 bucket (NVLink 5 / NVSwitch; the bucket
is tens of KB for the MLP, 6.7 MB for NatureCNN -- latency-bound, so exactly one collective, no bucketing).

For the hand-written update (clean_pufferl._DefaultMLPUpdate) the exchange is fused into the optimizer kernel over NVLink
peer memory (``PeerComm`` / csrc/peer.cu): no NCCL call per step, so the update is ONE CUDA graph at any world size.  The
fused recurrent update keeps torch's clip + Adam and takes the gradient mean alone over the same kind of peer memory
(``GradBucket.open_peer`` / ``peer_all_reduce_mean``, pb_peer_allreduce_mean), so it too is ONE graph on every rank.
"""
import ctypes as C
import os

import torch
import torch.distributed as dist


def init(backend=None):
    """Initialise torch.distributed from the torchrun environment (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_*)."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = 'nccl' if torch.cuda.is_available() else 'gloo'
        if backend == 'nccl':
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device('cuda', local))
        else:
            dist.init_process_group(backend)
    elif torch.cuda.is_available():
        torch.cuda.set_device(local)
    return rank, local, world


def shard(num_envs_total, rank, world):
    """Contiguous env shard of this rank: (env_index_offset, local num_envs)."""
    if num_envs_total % world != 0:
        raise ValueError('total num_envs must be divisible by the number of ranks')
    per = num_envs_total // world
    return rank * per, per


class GradBucket:
    """Flat fp32 gradient bucket: parameters' ``.grad`` are views into one buffer, so the all-reduce needs no
    pack/unpack copies."""

    def __init__(self, module):
        params = [p for p in module.parameters() if p.requires_grad]
        total = sum(p.numel() for p in params)
        self.flat = torch.zeros(total, dtype=torch.float32, device=params[0].device)
        off = 0
        for p in params:
            n = p.numel()
            p.grad = self.flat[off:off + n].view_as(p)
            off += n
        self.params = params
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        # PeerComm for the flat buffer (open_peer), or None: all_reduce_mean's NCCL call.  peer_tried: open_peer has run
        self.peer, self.peer_tried = None, False

    def open_peer(self):
        """Map a PeerComm over the flat buffer, with room for the 4-float KL payload after it (pb_peer_allreduce_mean), on
        every rank or on none.  Collective; once until close_peer.  -> None, or why peers are unavailable (NCCL then)."""
        self.peer_tried = True
        self.peer, msg = open_peer_comm((self.flat.numel() + 3) // 4 * 4 + 4, self.flat.device)
        return msg

    def close_peer(self):
        """Collective, like open_peer; the next open_peer maps a fresh communicator."""
        if self.peer is not None:
            self.peer.close()
        self.peer, self.peer_tried = None, False

    def zero(self):
        self.rebind()
        self.flat.zero_()

    def rebind(self):
        """optimizer.zero_grad(set_to_none=True) drops the views: re-attach them (cheap, no copies)."""
        off = 0
        for p in self.params:
            n = p.numel()
            if p.grad is None or p.grad.data_ptr() != self.flat.data_ptr() + off * 4:
                g = self.flat[off:off + n].view_as(p)
                if p.grad is not None:
                    g.copy_(p.grad)
                p.grad = g
            off += n

    def all_reduce_mean(self):
        self.rebind()
        if self.world > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
            self.flat.div_(self.world)

    def peer_all_reduce_mean(self, kl_in=None, kl_out=None):
        """all_reduce_mean over the peer buffers (open_peer): ONE kernel, no host call, so it can be captured; the same bits
        as all_reduce_mean on the same rank-order sum.  kl_in / kl_out (both or neither): device fp64 one-element tensors;
        kl_out <- kl_in summed over the ranks in rank order, carried by the same exchange."""
        from pufferlib_b200 import _native
        self.rebind()
        _native.check(_native.lib().pb_peer_allreduce_mean(C.byref(self.peer.struct), _native.ptr(self.flat), self.flat.numel(),
                                                           _native.ptr(kl_in), _native.ptr(kl_out), _native.stream_ptr()))


def broadcast_parameters(module, src=0):
    if dist.is_initialized() and dist.get_world_size() > 1:
        for p in module.parameters():
            dist.broadcast(p.data, src)
        for b in module.buffers():
            dist.broadcast(b.data, src)


class PeerComm:
    """NVLink peer-memory communicator for small flat fp32 buffers (csrc/peer.cu): every rank allocates one buffer with
    the C ABI (cudaMalloc + cudaIpcGetMemHandle), the 64-byte handles travel through torch.distributed once, every rank
    maps all peers.  ``struct`` is the pb_peer_comm the kernels take by value.  Single node only."""

    def __init__(self, capacity_floats, group=None):
        from pufferlib_b200 import _native
        if not (dist.is_initialized() and dist.get_world_size(group) > 1):
            raise RuntimeError('PeerComm needs an initialised process group with more than one rank')
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if self.world > 8:
            raise RuntimeError('PeerComm: at most 8 ranks (one NVSwitch node)')
        lib = _native.lib()
        self.capacity = (int(capacity_floats) + 3) & ~3      # multiple of 4 floats: both slots stay 16-byte aligned
        nbytes = lib.pb_peer_buffer_bytes(self.capacity)
        own, handle = C.c_void_p(), C.create_string_buffer(64)
        _native.check(lib.pb_peer_alloc(nbytes, C.byref(own), handle))
        self._own = own
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(handle.raw), group=group)
        self._opened = []
        bases = (C.c_void_p * 8)()
        for r, h in enumerate(handles):
            if r == self.rank:
                bases[r] = own.value
            else:
                p = C.c_void_p()
                _native.check(lib.pb_peer_open(C.create_string_buffer(h, 64), C.byref(p)))
                self._opened.append(p)
                bases[r] = p.value
        self.epoch = torch.zeros(1, dtype=torch.int64, device='cuda')
        self.struct = _native.PeerComm(world=self.world, rank=self.rank, base=bases, epoch=self.epoch.data_ptr(),
                                       capacity=self.capacity)
        torch.cuda.synchronize()
        dist.barrier(group=group)          # every buffer is zeroed and mapped before the first flag is raised

    def all_reduce_(self, flat):
        """In-place sum of a contiguous fp32 CUDA tensor over all ranks (one single-CTA kernel, graph-capturable)."""
        from pufferlib_b200 import _native
        assert flat.is_cuda and flat.dtype == torch.float32 and flat.is_contiguous() and flat.numel() <= self.capacity
        _native.check(_native.lib().pb_peer_allreduce(C.byref(self.struct), _native.ptr(flat), flat.numel(),
                                                      _native.stream_ptr()))
        return flat

    def close(self):
        from pufferlib_b200 import _native
        lib = _native.lib()
        torch.cuda.synchronize()
        for p in self._opened:
            lib.pb_peer_close(p)
        self._opened = []
        if self._own is not None:
            if dist.is_initialized():
                dist.barrier()             # nobody still has the buffer mapped / in use
            lib.pb_peer_free(self._own)
            self._own = None


def open_peer_comm(capacity_floats, device):
    """PeerComm(capacity_floats) on every rank, or None on every rank: all ranks agree through one all-reduce, and those
    that mapped their peers close them again when any rank could not.  -> (comm or None, why this rank failed or None)."""
    ok = torch.ones(1, device=device)
    comm, msg = None, None
    try:
        comm = PeerComm(capacity_floats)
    except Exception as e:           # every rank must take the same path: agree on it below
        msg = f'peer all-reduce unavailable ({type(e).__name__}: {e}); using NCCL'
        ok.zero_()
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if float(ok.item()) == 0.0:
        if comm is not None:
            comm.close()
        comm = None
    return comm, msg
