"""Staged peers for the gradient exchange of csrc/peer.cu on ONE device, shared by tests/test_gpu_peer_staged.py.  Not
collected by pytest (no test_ prefix).

pb_peer_comm is plain data: a world size, a rank, one device pointer per rank, a device epoch counter and a capacity.  The
kernels do not care where base[r] lives, so one process plays rank k of a world of W if it plays the other W - 1 ranks
BEFORE the launch: for the coming epoch e it writes rank r's gradient into slot e & 1 of buffer r and rank r's arrival
flags (value e) into buffer k.  The kernel then copies its own gradient into its slot, raises its own flags in all W
buffers, finds every peer flag already there and sums the W slots in rank order.  It never waits.

The kernels' waits are bounded by a device trap, which is fatal to the CUDA context.  So every launch that contains a wait
goes through `StagedPeers.exchange` (or `replay` for a captured graph): it stages with stream-ordered torch writes on
the launch stream, checks the device epoch against its own count, and asserts from its own bookkeeping that every flag the
kernel will poll was written for this epoch.  Nothing here exercises the wait, a missing peer or two kernels that wait on
each other.  (Each CTA also polls its own rank's flag in its own buffer, the one it has just raised; staging cannot stand in
for that one, so a kernel change that moves the flag store makes the kernel wait: check such a change on the CPU first.)

`StagedPeers` also keeps a mirror of what all W buffers must hold after every call (the protocol restated with torch
indexing); `check_buffers` compares whole buffers with it bit for bit, so a stray store anywhere in a header, a slot tail
or the other parity's slot shows up.
"""
import ctypes as C

import torch

from pufferlib_b200 import _native

HEADER_WORDS = 128          # 1024-byte header = 128 uint64: the flag of source rank r, slice b is word 16 r + b
HEADER_FLOATS = 256
SLICES = 16


def gradients(n, world, seed, dev, scale=1.0):
    """One fp32 gradient of n elements per rank: mixed sign, magnitudes log-uniform over 1e-3 .. 1e3 (times `scale`), so the
    order of the fp32 additions over the ranks changes the bits of the sum."""
    gen = torch.Generator(device='cpu').manual_seed(seed)
    mag = 10.0 ** (6.0 * torch.rand(world, n, generator=gen, dtype=torch.float64) - 3.0)
    sign = torch.where(torch.rand(world, n, generator=gen) < 0.5, -1.0, 1.0)
    return (mag * sign * scale).float().to(dev)


def rank_order_sum(g):
    """What the kernels compute: s = 0; s += g[0]; s += g[1]; ... in fp32, one rounding per addition."""
    s = torch.zeros_like(g[0])
    for r in range(g.shape[0]):
        s = s + g[r]
    return s


def bits(t):
    return t.contiguous().view(torch.int32)


def slice_bounds(n):
    """Element range of each of the 16 slices of the sliced exchange: chunks of ceil(n / 16) rounded up to 4 floats; the
    trailing slices of a short buffer are empty."""
    chunk = (-(-n // SLICES) + 3) // 4 * 4
    return [(min(b * chunk, n), min((b + 1) * chunk, n)) for b in range(SLICES)]


class StagedPeers:
    """W peer buffers on one device with this process as rank `rank`.  sliced: the 16-CTA kernels (flags 16 r + b), else
    the one-CTA kernel (flag 16 r)."""

    def __init__(self, world, rank, capacity, dev, sliced):
        assert 2 <= world <= 8 and 0 <= rank < world and capacity >= 1
        self.world, self.rank, self.capacity, self.sliced, self.dev = world, rank, capacity, sliced, dev
        nbytes = _native.lib().pb_peer_buffer_bytes(capacity)
        assert nbytes == 1024 + 8 * capacity
        # every slot element starts as a NaN whose payload names its buffer and position: a canary read into a sum is a NaN
        self.bufs = []
        for r in range(world):
            buf = torch.zeros(nbytes // 8, dtype=torch.int64, device=dev)
            idx = torch.arange(2 * capacity, dtype=torch.int32, device=dev)
            buf[HEADER_WORDS:].view(torch.int32).copy_(0x7FC00000 | (((r + 1) << 18) ^ (idx & 0x3FFFF)))
            self.bufs.append(buf)
        self.mirror = [b.clone() for b in self.bufs]
        self.epoch_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        self.epoch = 0                      # host count of finished exchanges: the device counter must agree
        base = (C.c_void_p * 8)()
        for r in range(world):
            base[r] = self.bufs[r].data_ptr()
        self.struct = _native.PeerComm(world=world, rank=rank, base=base, epoch=self.epoch_dev.data_ptr(), capacity=capacity)
        self.flag_slices = range(SLICES) if sliced else range(1)

    def slot(self, buf, parity):
        """Slot `parity` of a buffer (or of its mirror) as floats."""
        off = HEADER_FLOATS + parity * self.capacity
        return buf.view(torch.float32)[off:off + self.capacity]

    def _flag_words(self, r):
        return [16 * r + b for b in self.flag_slices]

    def _stage(self, e, peer_grads, n, flag_value):
        """Play the peers for epoch e: their gradients into their slots, their flags (flag_value >= e) into the own buffer.
        -> the set of (rank, slice) flags written."""
        k = self.rank
        staged = set()
        for r in range(self.world):
            if r == k:
                continue
            for buf in (self.bufs[r], self.mirror[r]):
                self.slot(buf, e & 1)[:n].copy_(peer_grads[r])
            words = torch.tensor(self._flag_words(r), device=self.dev)
            self.bufs[k][words] = flag_value
            self.mirror[k][words] = flag_value
            staged.update((r, b) for b in self.flag_slices)
        return staged

    def _polled(self):
        """The flags the kernel's CTAs poll in the own buffer, besides the ones it raises itself."""
        return {(r, b) for r in range(self.world) if r != self.rank for b in self.flag_slices}

    def exchange(self, flat, peer_grads, launch, advances=True):
        """Stage the peers for the next epoch, then launch(comm) on the current stream; launch must sum `flat` (n floats, the
        own gradient) in place.  peer_grads: [W, n], row `rank` unused.  advances: whether what `launch` enqueues advances the
        epoch counter (pb_peer_allreduce_parts alone does not: the pb_clip_adam_parts call after it does).  -> the epoch."""
        n = flat.numel()
        assert n <= self.capacity and peer_grads.shape == (self.world, n)
        assert int(self.epoch_dev.item()) == self.epoch, 'device epoch out of step with the staging: refusing to launch'
        e = self.epoch + 1
        staged = self._stage(e, peer_grads, n, e)
        assert staged == self._polled(), 'a flag the kernel polls was not staged'
        # what the kernel itself must leave: the own gradient in the own slot, the own flags in every buffer
        self.slot(self.mirror[self.rank], e & 1)[:n].copy_(flat)
        for r in range(self.world):
            self.mirror[r][torch.tensor(self._flag_words(self.rank), device=self.dev)] = e
        launch(self.struct)
        if advances:
            self.epoch = e
        return e

    def advanced(self):
        """A later kernel in the stream advanced the epoch counter (pb_clip_adam_parts with peer_epoch)."""
        self.epoch += 1

    def capture(self, enqueue):
        """enqueue(comm) inside a CUDA graph capture (which runs nothing) -> the graph; run it with `replay` only."""
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(graph):
            enqueue(self.struct)
        return graph

    def replay(self, graph, peer_grads_by_parity, n, steps):
        """Replay a captured graph of `steps` exchanges.  Staged first: both slots of every peer (one gradient set per parity,
        [2][W, n]) and every peer flag at the last epoch the replay reaches (a flag only has to be >= the epoch polled for)."""
        assert int(self.epoch_dev.item()) == self.epoch, 'device epoch out of step with the staging: refusing to replay'
        last = self.epoch + steps
        for parity in (0, 1):
            staged = self._stage(parity, peer_grads_by_parity[parity], n, last)
            assert staged == self._polled(), 'a flag the kernel polls was not staged'
        graph.replay()
        self.epoch = last

    def check_epoch(self):
        got = int(self.epoch_dev.item())
        assert got == self.epoch, f'epoch counter {got}, expected {self.epoch}'

    def check_buffers(self):
        """Every byte of all W buffers against the mirror."""
        for r in range(self.world):
            if not torch.equal(self.bufs[r], self.mirror[r]):
                bad = (self.bufs[r] != self.mirror[r]).nonzero().flatten()
                head = [int(w) for w in bad if w < HEADER_WORDS]
                body = [int(w) - HEADER_WORDS for w in bad if w >= HEADER_WORDS]
                raise AssertionError(
                    f'buffer {r} (own rank {self.rank}, epoch {self.epoch}): header words {head[:8]} and float pairs '
                    f'{body[:8]} of the slots (capacity {self.capacity}) differ from the protocol; '
                    f'got {[hex(int(self.bufs[r][w])) for w in bad[:4]]}, expected {[hex(int(self.mirror[r][w])) for w in bad[:4]]}')
