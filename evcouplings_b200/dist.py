"""
Multi-process plumbing (one process per GPU, torch.distributed).  The PLM path shards naturally:

* PLL objective/gradient -- sequences are independent units: contiguous blocks of sequences per rank,
  parameters replicated, ONE all-reduce(sum) of the gradient (+ 8 bytes of -loglk) per evaluation;
* Hamming reweighting   -- the upper-triangular 128x128 pair tiles are split in contiguous ranges per
  rank (every unordered pair is visited exactly once globally), then all-reduce(sum) of int32 counters.

Backend is whatever the process group was created with: "nccl" on GPUs (NVLink/NVSwitch), "gloo" in the
CPU-only tests of this logic.
"""


def shard_bounds(n, world, rank):
    """Contiguous block partition of n items over `world` ranks (sizes differ by <= 1)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class Collective(object):
    """Thin wrapper over torch.distributed that degrades to a no-op for a single process."""

    def __init__(self, group=None, standalone=False):
        import torch.distributed as dist
        self.dist = dist
        self.group = group
        if not standalone and dist.is_available() and dist.is_initialized():
            self.rank = dist.get_rank(group)
            self.world = dist.get_world_size(group)
        else:
            self.rank, self.world = 0, 1

    def all_reduce_sum(self, tensor):
        if self.world > 1:
            self.dist.all_reduce(tensor, op=self.dist.ReduceOp.SUM, group=self.group)
        return tensor

    def all_reduce_max(self, tensor):
        if self.world > 1:
            self.dist.all_reduce(tensor, op=self.dist.ReduceOp.MAX, group=self.group)
        return tensor

    def all_gather(self, tensor):
        """Every rank's ``tensor`` (same shape and dtype on all ranks), as a list in rank order."""
        if self.world == 1:
            return [tensor]
        out = [tensor.new_empty(tensor.shape) for _ in range(self.world)]
        self.dist.all_gather(out, tensor, group=self.group)
        return out

    def barrier(self):
        if self.world > 1:
            self.dist.barrier(group=self.group)


def hamming_tile_coords(idx, T):
    """(R, C) of linear upper-triangular tile index idx (row-major over R, C >= R), T tiles per side.
    Host-side twin of tile_from_index in csrc/hamming.cu."""
    r = 0
    # offset(R) = R*T - R(R-1)/2
    lo, hi = 0, T - 1
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if mid * T - mid * (mid - 1) // 2 <= idx:
            lo = mid
        else:
            hi = mid - 1
    r = lo
    return r, r + (idx - (r * T - r * (r - 1) // 2))
