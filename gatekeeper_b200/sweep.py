"""Sharded audit sweep: every rank reviews its own contiguous range of the cluster's objects and the violation
bitmaps are all-gathered once (SURVEY.md 8(e)); per-constraint totals are all-reduced.

Objects are independent units, so there is no data-path collective besides that final exchange.  On GPUs the
kernel writes straight into torch-owned device buffers on torch's current stream and NCCL gathers them; the
same function runs under `gloo` with host tensors (tests use the CPU test backend there).
"""
from __future__ import annotations

import os
from typing import Optional, Tuple


class _PeerExchange:
    """Symmetric (peer-mapped) receive buffers: buffers[k] is this rank's k-th buffer, bases[k][q] the device address of
    rank q's k-th buffer as mapped into this process."""

    def __init__(self, torch, world, slot_i32, device):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        self.rank = dist.get_rank()
        self.buffers, self.handles, self.bases = [], [], []
        for _ in range(2):
            buf = symm.empty(world * slot_i32, dtype=torch.int32, device=device)
            buf.zero_()
            hdl = symm.rendezvous(buf, dist.group.WORLD)
            self.buffers.append(buf)
            self.handles.append(hdl)
            self.bases.append([int(p) for p in hdl.buffer_ptrs])
        torch.cuda.synchronize()
        dist.barrier()


def shard_range(n_total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous object range [lo, hi) of a rank (GPU g gets objects [g*N/G, (g+1)*N/G))."""
    return n_total * rank // world, n_total * (rank + 1) // world


class ShardedSweep:
    """Holds a resident batch (this rank's shard) and the torch buffers for the exchange.

    The per-constraint totals ride at the tail of the bitmap shard, so the step's exchange is ONE collective (an
    all-gather); the totals of all ranks are then summed locally."""

    def __init__(self, drv, resident_batch, n_local: int, n_constraints: int, device, world: int = 1):
        import torch
        self.torch = torch
        self.drv, self.rb, self.n, self.C = drv, resident_batch, n_local, n_constraints
        self.words = max(1, (n_constraints + 31) // 32)
        self.world = world
        self.device = device
        self.on_gpu = device.type == "cuda"
        cmax = max(1, n_constraints)
        bitmap_i32 = n_local * self.words
        pad = bitmap_i32 % 2                                   # the int64 totals that follow must be 8-byte aligned
        self._tot_off = bitmap_i32 + pad
        self._send = torch.zeros(self._tot_off + 4 * cmax, dtype=torch.int32, device=device)
        self.viol = self._send[:bitmap_i32].view(n_local, self.words)
        self.tot_local = self._send[self._tot_off:].view(torch.int64).view(2, cmax)     # [violations, matcher errors] x constraint
        self.tot = self.tot_local if world == 1 else torch.zeros((2, cmax), dtype=torch.int64, device=device)
        self.err = torch.zeros((n_local, self.words), dtype=torch.int32, device=device)
        self._recv = torch.zeros(world * self._send.numel(), dtype=torch.int32, device=device) if world > 1 else None
        self.gathered = None
        # Fused exchange over NVLink peer memory (GPUs only): two symmetric receive buffers used alternately, so that a
        # fast rank's next kernel never overwrites what a slow rank is still reading; one device-side barrier per step.
        self.p2p = None
        if world > 1 and self.on_gpu and os.environ.get("GK_P2P", "1") != "0":
            try:
                self.p2p = _PeerExchange(torch, world, self._send.numel(), device)
            except Exception as e:                      # no peer access / symmetric memory: the NCCL all-gather remains
                self.p2p_error = repr(e)
                self.p2p = None
        self._step = 0

    def evaluate(self, enforcement_point: str, stream=None):
        """One pass of the hot path over the shard: kernel -> (viol, err, totals) in this rank's buffers."""
        torch = self.torch
        if self.on_gpu and self.p2p is not None:
            st = stream if stream is not None else torch.cuda.current_stream()
            px = self.p2p
            self.rb.eval_device_peers(enforcement_point, px.bases[self._step & 1], px.rank, self._send.numel(), self._tot_off, self.tot_local.shape[1],
                                      self.err.data_ptr(), self.tot_local[0].data_ptr(), self.tot_local[1].data_ptr(), st.cuda_stream)
        elif self.on_gpu:
            st = stream if stream is not None else torch.cuda.current_stream()
            self.rb.eval_device(enforcement_point, self.viol.data_ptr(), self.err.data_ptr(), self.tot_local[0].data_ptr(),
                                self.tot_local[1].data_ptr(), st.cuda_stream)
        else:
            r = self.rb.eval(enforcement_point)
            self.viol.copy_(torch.from_numpy(r.viol_bits.view("int32")))
            self.err.copy_(torch.from_numpy(r.err_bits.view("int32")))
            self.tot_local.zero_()
            self.tot_local[0, :self.C] = torch.tensor(r.totals, dtype=torch.int64)
            self.tot_local[1, :self.C] = torch.tensor(r.err_totals, dtype=torch.int64)

    def exchange(self):
        """The one collective of the path: all-gather of (bitmap shard | totals); totals are summed over ranks locally."""
        if self.world == 1:
            return self.viol, self.tot
        if self.p2p is not None:
            # every rank's kernel has written its shard (and totals) into everybody's buffer: wait for all of them
            self.p2p.handles[self._step & 1].barrier(channel=0)
            recv = self.p2p.buffers[self._step & 1].view(self.world, -1)
            self._step += 1
        else:
            import torch.distributed as dist
            dist.all_gather_into_tensor(self._recv, self._send)
            recv = self._recv.view(self.world, -1)
        bitmap_i32 = self.n * self.words
        self.gathered = recv[:, :bitmap_i32]                                         # [world, n_local * words] (a view)
        self.tot.copy_(recv[:, self._tot_off:].contiguous().view(self.torch.int64).view(self.world, 2, -1).sum(0))
        return self.gathered, self.tot       # row g = rank g's bitmap shard, n_local * words int32 (no copy is made)

    def step(self, enforcement_point: str):
        self.evaluate(enforcement_point)
        return self.exchange()


class ShardedAudit:
    """The audit's constraint status over a sharded sweep: every rank folds its own pages into an AuditRun
    (add_batch_ordered: the lazy path for any mix of kinds), then the runs' exports are all-gathered and merged in rank
    order, so that every rank holds the report one run over all shards in rank order would give.

    The exchange is two collectives on the default group (gloo or NCCL): the export sizes, then the exports padded to the
    largest as uint8 tensors."""

    def __init__(self, drv, violations_limit: int = 0, msg_size: int = 0, device=None):
        from gatekeeper_b200 import driver as D
        self.drv, self.limit, self.msg_size = drv, violations_limit, msg_size
        self.run = D.AuditRun(drv, violations_limit, msg_size)
        self.device = device
        self.merged = None
        self.timing = {}

    def add_batch(self, rb, enforcement_point: str):
        self.run.add_batch_ordered(rb, enforcement_point)

    def exchange(self) -> dict:
        """All-gather every rank's run, merge them in rank order; returns the merged report (the same on every rank)."""
        import time
        import torch
        import torch.distributed as dist
        from gatekeeper_b200 import driver as D
        dev = self.device if self.device is not None else torch.device("cpu")
        world = dist.get_world_size() if dist.is_initialized() else 1
        t0 = time.perf_counter()
        mine = self.run.export()
        t1 = time.perf_counter()
        if world == 1:
            parts = [mine]
        else:
            size = torch.tensor([len(mine)], dtype=torch.int64, device=dev)
            sizes = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
            dist.all_gather(sizes, size)
            lens = [int(s.item()) for s in sizes]
            pad = max(lens)
            send = torch.zeros(pad, dtype=torch.uint8)
            send[:len(mine)] = torch.frombuffer(bytearray(mine), dtype=torch.uint8)
            send = send.to(dev)
            recv = [torch.zeros(pad, dtype=torch.uint8, device=dev) for _ in range(world)]
            dist.all_gather(recv, send)
            parts = [bytes(r[:k].cpu().numpy().tobytes()) for r, k in zip(recv, lens)]
        t2 = time.perf_counter()
        merged = D.AuditRun(self.drv, self.limit, self.msg_size)
        for p in parts:
            merged.merge(p)
        t3 = time.perf_counter()
        if self.merged is not None:
            self.merged.close()
        self.merged = merged
        self.timing = {"export_ms": (t1 - t0) * 1e3, "exchange_ms": (t2 - t1) * 1e3, "merge_ms": (t3 - t2) * 1e3, "bytes": sum(len(p) for p in parts)}
        return merged.report()
