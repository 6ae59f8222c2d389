"""Multi-GPU plumbing for the batch-sharded forward (SURVEY.md 8(e)): one process per GPU, samples are independent,
weights / graphs are replicated, and the only communication is ONE gather of the per-rank outputs at the loss boundary
(or, with the fused loss, one scalar: losses.py).  torch.distributed is the rendezvous and the fallback transport.

`BoundaryGather` is that one collective, built so that it does not take SMs away from the persistent chain kernels
(they hold every SM with 227 KB of shared memory, so an NCCL kernel issued beside them only runs in the gaps between
them and stalls the statically scheduled tiles of the next kernel -- measured in round 1: no overlap at all):

  * mode "fused"     `gather.forward(model, features)`: the chain kernel that produces the forecast stores every tile of it, as it
                     leaves the tensor cores, into the gather buffer of EVERY GPU -- one multimem.st per value to the NVLink
                     multicast alias of the symmetric buffer (the NVSwitch replicates it), or one store per peer mapping where
                     multicast is unavailable (csrc/gw_tc3.cu out_mode, gw_plan_set_output_peers).  Compute and collective are one
                     kernel; two symmetric-memory barriers (a few microseconds) order it.  No separate transfer exists.
  * mode "p2p_copy"  every rank owns a symmetric-memory gather buffer (torch symmetric memory: cuMem allocations mapped
                     into every peer over NVLink).  A rank's shard is pushed into each peer's buffer by the COPY ENGINES
                     (device-to-device cudaMemcpyAsync into the peer mapping, no kernel), on a side stream, followed by the
                     symmetric-memory barrier; the next step's forward runs underneath.
  * mode "nccl"      all_gather_into_tensor on the side stream (fallback when symmetric memory is unavailable).
  * gloo / CPU       `all_gather_batch` (tests).
"""

from __future__ import annotations

import torch
import torch.distributed as dist


def shard_range(total_batch: int, rank: int, world: int):
    """Contiguous, balanced [start, stop) of the global batch owned by `rank` (earlier ranks take the remainder)."""
    base, rem = divmod(total_batch, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def all_gather_batch(y: torch.Tensor, total_batch: int, group=None) -> torch.Tensor:
    """Gathers per-rank outputs [b_r, ...] into [total_batch, ...] in rank order; shards may differ by one sample."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_range(total_batch, r, world) for r in range(world)]
    assert y.shape[0] == sizes[rank][1] - sizes[rank][0], "local shard does not match shard_range"
    bmax = max(b - a for a, b in sizes)
    if all(b - a == bmax for a, b in sizes):
        out = torch.empty((world * bmax,) + tuple(y.shape[1:]), dtype=y.dtype, device=y.device)
        dist.all_gather_into_tensor(out, y.contiguous(), group=group)
        return out
    pad = torch.zeros((bmax,) + tuple(y.shape[1:]), dtype=y.dtype, device=y.device)
    pad[: y.shape[0]] = y
    buf = torch.empty((world * bmax,) + tuple(y.shape[1:]), dtype=y.dtype, device=y.device)
    dist.all_gather_into_tensor(buf, pad, group=group)
    return torch.cat([buf[r * bmax : r * bmax + (b - a)] for r, (a, b) in enumerate(sizes)], dim=0)


def max_over_ranks(value: float, device, group=None) -> float:
    t = torch.tensor([float(value)], device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return float(t.item())


class BoundaryGather:
    """gather = BoundaryGather(total_batch, device); out = gather(y); ...; gather.wait(); use(out)

    `out` is the [total_batch, ...] gather of every rank's `y` in rank order.  The transfer runs on a side stream; the
    calling stream is not blocked until `wait()` (or the next call that reuses the same buffer, two calls later), so the
    next forward overlaps it.  `overlap=False` makes the call itself wait."""

    def __init__(self, total_batch: int, device, group=None, mode: str = "auto"):
        self.total = int(total_batch)
        self.device = torch.device(device)
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.ranges = [shard_range(self.total, r, self.world) for r in range(self.world)]
        self.mode = mode
        self.side = torch.cuda.Stream(self.device) if self.device.type == "cuda" else None
        self._bufs = None  # [2] local gather buffers
        self._peers = None  # [2][world] peer mappings of the same buffers (p2p_copy)
        self._hdl = None
        self._done = [None, None]
        self._i = 0
        self.fallback_reason = None

    def _setup(self, y):
        shape = (self.total,) + tuple(y.shape[1:])
        want = self.mode
        if self.device.type != "cuda":
            self.mode = "gloo"
            return
        if want in ("auto", "fused", "fused_peer", "p2p_copy"):
            try:
                import torch.distributed._symmetric_memory as symm_mem

                pg = self.group if self.group is not None else dist.group.WORLD
                self._bufs, self._hdl, self._peers, self._fused = [], [], [], []
                for _ in range(2):
                    t = symm_mem.empty(shape, dtype=y.dtype, device=self.device)
                    h = symm_mem.rendezvous(t, pg)
                    self._bufs.append(t)
                    self._hdl.append(h)
                    self._peers.append([h.get_buffer(r, shape, y.dtype) for r in range(self.world)])
                    # aliases of this rank's buffer for the in-kernel stores: (mode, byte deltas from the local address)
                    ptrs = [int(v) for v in h.buffer_ptrs]
                    mc = int(getattr(h, "multicast_ptr", 0) or 0)
                    if mc and want != "fused_peer" and self.world <= 8:
                        self._fused.append((1, [mc - ptrs[self.rank]]))
                    elif self.world <= 8:
                        self._fused.append((2, [ptrs[r] - ptrs[self.rank] for r in range(self.world)]))
                # "auto" takes the copy engines: their transfer overlaps the next forward, while in-kernel stores of the 78-wide
                # (312-byte, 8-byte aligned) forecast rows lengthen the last chain
                self.mode = "fused" if want in ("fused", "fused_peer") and len(self._fused) == 2 else "p2p_copy"
                return
            except Exception as e:  # no symmetric memory on this box / build: NCCL on the side stream
                if want != "auto":
                    raise
                self.fallback_reason = f"{type(e).__name__}: {e}"
        self._bufs = [torch.empty(shape, dtype=y.dtype, device=self.device) for _ in range(2)]
        self.mode = "nccl"

    def __call__(self, y: torch.Tensor, overlap: bool = True) -> torch.Tensor:
        a, b = self.ranges[self.rank]
        assert y.shape[0] == b - a, "local shard does not match shard_range"
        if self._bufs is None and self.mode != "gloo":
            self._setup(y)
        if self.mode == "gloo":
            return all_gather_batch(y, self.total, self.group)
        if self.mode == "fused":  # called with a finished tensor: the copy-engine path moves it (same buffers)
            return self._copy_gather(y, overlap)
        return self._copy_gather(y, overlap)

    def forward(self, model, features: torch.Tensor, overlap: bool = True) -> torch.Tensor:
        """model(features) on this rank's shard, gathered over all ranks: [total_batch, N, F].  In mode "fused" the forward
        itself writes into every GPU's gather buffer (no transfer after it); otherwise forward, then the gather."""
        if self._bufs is None and self.mode not in ("gloo",):
            B, N = features.shape[0], features.shape[1]
            self._setup(torch.empty((B, N, model.output_dim), dtype=torch.float32, device=features.device))
        if self.mode != "fused":
            return self(model(features), overlap=overlap)
        # (selectable with mode="fused" / "fused_peer"; see _setup for the measured trade-off)
        a, b = self.ranges[self.rank]
        assert features.shape[0] == b - a, "local shard does not match shard_range"
        k = self._i & 1
        self._i += 1
        h = self._hdl[k]
        mode, deltas = self._fused[k]
        h.barrier(channel=0)  # every rank has finished with buffer k (its use two calls ago) before anybody stores into it
        model.forward_into(features, self._bufs[k][a:b], peers=(mode, deltas))
        h.barrier(channel=1)  # the stores of every rank have landed in every buffer
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._done[k] = ev
        return self._bufs[k]

    def _copy_gather(self, y: torch.Tensor, overlap: bool = True) -> torch.Tensor:
        a, b = self.ranges[self.rank]
        k = self._i & 1
        self._i += 1
        cur = torch.cuda.current_stream(self.device)
        if self._done[k] is not None:
            cur.wait_event(self._done[k])  # the gather that used this buffer two calls ago has landed (and was consumed in stream order)
        ready = torch.cuda.Event()
        ready.record(cur)
        self.side.wait_event(ready)
        y = y.contiguous()
        with torch.cuda.stream(self.side):
            if self.mode in ("p2p_copy", "fused"):
                h = self._hdl[k]
                h.barrier(channel=0)  # every rank is past the forward of this step: nobody still reads buffer k
                for d in range(self.world):  # own slot first, then the peers in ring order (spreads the NVSwitch ports)
                    r = (self.rank + d) % self.world
                    self._peers[k][r][a:b].copy_(y, non_blocking=True)  # copy engine; r == rank is the local slot
                h.barrier(channel=1)  # every shard has landed in every buffer
            else:
                if all(e - s == b - a for s, e in self.ranges):
                    dist.all_gather_into_tensor(self._bufs[k], y, group=self.group)
                else:
                    self._bufs[k].copy_(all_gather_batch(y, self.total, self.group))
            ev = torch.cuda.Event()
            ev.record(self.side)
        y.record_stream(self.side)
        self._done[k] = ev
        if not overlap:
            cur.wait_event(ev)
        return self._bufs[k]

    def wait(self):
        """Makes the calling stream wait for every gather issued so far."""
        if self.side is None:
            return
        cur = torch.cuda.current_stream(self.device)
        for ev in self._done:
            if ev is not None:
                cur.wait_event(ev)
