"""NVLink peer-memory collectives of the step (`csrc/comm.cu`): host side.

One symmetric allocation per rank (torch.distributed._symmetric_memory: cuMem + handle
exchange; PyTorch is the allocator / rendezvous plumbing, the data path is our kernels),
carved into

  bn      NSLOT x world x SLOT_BYTES   one-shot SyncBN exchanges ([2C] doubles per rank)
  gather  per channel: world x capacity  all-gather regions ('z': embeddings, 'lse')
  flags   u64 words

`PeerComm.create(group)` returns None when peer memory cannot be set up (single rank, no
P2P, SIMCLR_COMM=nccl): the callers then use torch.distributed / NCCL for the same
collectives.  Either path computes the same values; the peer path is what the scaling
numbers are measured with.
"""
import collections
import os

import torch
import torch.distributed as dist

from ._lib import lib, stream_ptr

NSLOT = 4
MAX_CHANNELS = 8192                      # widest BatchNorm (ResNet 2x / 4x heads): 2*C doubles per slot
SLOT_BYTES = 2 * MAX_CHANNELS * 8
GATHER_CHANNELS = {'z': 4 << 20, 'lse': 256 << 10}     # bytes per rank


Layout = collections.namedtuple('Layout', 'bn_off gather_off bn_flag_off gather_flag_off total')


def layout(world):
    """Byte offsets of the regions of one rank's allocation for `world` ranks (the same on every rank): the bn
    slots, the gather region of each channel, the bn flag words, the flag words of each channel, and the total
    size (a whole number of 4 KiB pages)."""
    off = 0
    bn_off = off; off += NSLOT * world * SLOT_BYTES
    gather_off = {}
    for name, cap in GATHER_CHANNELS.items():
        gather_off[name] = off; off += world * cap
    bn_flag_off = off; off += NSLOT * world * 8
    gather_flag_off = {}
    for name in GATHER_CHANNELS:
        gather_flag_off[name] = off; off += world * 8
    return Layout(bn_off, gather_off, bn_flag_off, gather_flag_off, (off + 4095) // 4096 * 4096)


def gather_fits(channel, nbytes):
    """Whether a tensor of `nbytes` per rank can go through the peer-memory gather `channel`; a larger one, or
    one that is not a 16-byte multiple, is gathered through NCCL."""
    return 0 < nbytes <= GATHER_CHANNELS[channel] and nbytes % 16 == 0


class PeerComm:
    def __init__(self, rank, world, buf, peers_dev, handle=None):
        """`buf`: this rank's zeroed allocation of `layout(world).total` bytes; `peers_dev`: the address of a
        device array of the `world` ranks' `buf` base pointers, in rank order.  `create` makes both in symmetric
        memory (`handle` keeps that rendezvous alive)."""
        self.rank, self.world = rank, world
        self.buf, self.peers_dev, self.handle = buf, peers_dev, handle
        self.device = buf.device
        self.slot_bytes = SLOT_BYTES
        self.bn_off, self.gather_off, self.bn_flag_off, self.gather_flag_off, self.total = layout(world)
        assert buf.numel() >= self.total, (buf.numel(), self.total)
        device = self.device
        # sequence numbers (start at 1: flag words start at 0) and CTA arrival counters, local memory
        # [sequence, nanoseconds spent waiting for peers] per channel
        self.bn_seq = torch.tensor([1, 0], dtype=torch.int64, device=device)
        self.gather_seq = {n: torch.tensor([1, 0], dtype=torch.int64, device=device) for n in GATHER_CHANNELS}
        self.gather_arrive = {n: torch.zeros(1, dtype=torch.int32, device=device) for n in GATHER_CHANNELS}

    @staticmethod
    def _symmetric(group, device):
        import torch.distributed._symmetric_memory as symm
        group = group if group is not None else dist.group.WORLD
        world = dist.get_world_size(group)
        buf = symm.empty(layout(world).total, dtype=torch.uint8, device=device)
        handle = symm.rendezvous(buf, group.group_name)
        buf.zero_()
        comm = PeerComm(dist.get_rank(group), world, buf, int(handle.buffer_ptrs_dev), handle)
        torch.cuda.synchronize(device)
        dist.barrier(group)             # nobody pushes before every buffer is zeroed
        torch.cuda.synchronize(device)
        return comm

    @staticmethod
    def create(group=None, device=None):
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) < 2:
            return None
        if os.environ.get('SIMCLR_COMM', 'peer') == 'nccl':
            return None
        device = device or torch.device('cuda', torch.cuda.current_device())
        try:
            return PeerComm._symmetric(group, device)
        except Exception as exc:      # no P2P / symmetric memory on this system: NCCL carries the collectives
            if os.environ.get('SIMCLR_COMM') == 'peer_required':
                raise
            import warnings
            warnings.warn('simclr_b200: peer-memory collectives unavailable (%r); using NCCL' % (exc,))
            return None

    def wait_ns(self):
        """Nanoseconds this rank has spent inside the exchange kernels waiting for its peers, since creation
        (device counters: a synchronising read).  The slowest rank of a step waits ~0; the others wait for it."""
        return int(self.bn_seq[1].item()) + sum(int(t[1].item()) for t in self.gather_seq.values())

    # -- fused SyncBN exchanges ----------------------------------------------------
    def _bn_args(self):
        return (self.peers_dev, self.rank, self.world, self.bn_off, self.bn_flag_off, NSLOT, SLOT_BYTES, self.bn_seq)

    def bn_finalize(self, sums, count_local, gamma, beta, eps, momentum, mm, mv, mean, rstd, scale, shift, C):
        lib.comm_bn_finalize(sums, float(count_local), gamma, beta, eps, momentum, mm, mv, mean, rstd, scale, shift, C,
                             *self._bn_args(), stream_ptr())

    def bn_bwd_coef(self, sums, count_local, mean, rstd, gamma, coef, dgamma, dbeta, C):
        lib.comm_bn_bwd_coef(sums, float(count_local), mean, rstd, gamma, coef, dgamma, dbeta, C,
                             *self._bn_args(), stream_ptr())

    # -- all-gather ------------------------------------------------------------------
    def all_gather(self, t, channel):
        """[...] -> [world, ...] (rank-major), a view of the local gather region of `channel`."""
        t = t.contiguous()
        nbytes = t.numel() * t.element_size()
        if not gather_fits(channel, nbytes):
            raise ValueError('all_gather(%s): %d bytes per rank (need a 16-byte multiple <= %d)'
                             % (channel, nbytes, GATHER_CHANNELS[channel]))
        off = self.gather_off[channel]
        lib.comm_all_gather(t, nbytes, self.peers_dev, self.rank, self.world, off, self.gather_flag_off[channel],
                            nbytes, self.gather_seq[channel], self.gather_arrive[channel], stream_ptr())
        return self.buf[off:off + self.world * nbytes].view(t.dtype).view((self.world,) + tuple(t.shape))
