"""Track sharding and the per-iteration all-reduce of the reduced camera system (SURVEY.md section 8e).

The reference has no distributed code (SURVEY.md section 2.2); this is new.  One process per GPU:
every rank holds all S cameras and a contiguous slice of the N tracks; point blocks, coupling blocks
and the Schur products are local; the reduced system [D x Dpad | rhs | diag | g] is summed across
ranks once per LM iteration (NCCL over NVLink / NVSwitch), after which every rank factors the same
small system redundantly and back-substitutes its own points.  A second, tiny all-reduce carries the
candidate cost and gradient so all ranks take the same accept/reject decision.

With linear_solver_type="ITERATIVE_SCHUR" nothing dense is reduced: AllReduceHook (without a fabric) sums the
assembled right-hand side, diagonal, gradient, preconditioner accumulators and camera records once per LM iteration and
one D-vector, the Schur part of the CG's matrix-vector product, per CG iteration; the CG's scalars are fixed-order
sums of summed data, so every rank takes the same CG decisions and makes the same sequence of hook calls.
"""
from __future__ import annotations

import ctypes

import torch
import torch.distributed as dist

from . import _lib


def shard_range(N: int, rank: int, world: int, multiple: int = 16):
    """Contiguous [lo, hi) slice of the track axis for `rank`; slices are multiples of `multiple`
    (TMA alignment) except the last.  Mirrors torch.chunk's contiguous split of
    vggsfm/utils/triangulation.py:721-733."""
    per = (N + world - 1) // world
    per = (per + multiple - 1) // multiple * multiple
    lo = min(N, rank * per)
    hi = min(N, lo + per)
    return lo, hi


class FabricBuffer:
    """Reduced-system buffer in symmetric (peer-mapped, NVSwitch-multicast) memory for the fused reduction
    (include/vggsfm_b200.h: vgg_ba_fabric).  The tensor-core SYRK's epilogue REDs every 128-row block of the lower
    triangle into its owner's copy over NVLink (reduce-scatter), every rank then pulls the blocks it does not own
    (csrc/fabric.cu), and the barriers / small all-reduces of the LM loop are kernels on the same allocation -- no NCCL
    call and no host callback inside the loop.  ``ok`` is False when the group lacks multicast or a peer table for
    2..8 ranks; AllReduceHook then reduces through NCCL instead."""

    def __init__(self, S: int, model: int, mode: int, device, group=None):
        import torch.distributed._symmetric_memory as symm_mem
        group = group if group is not None else dist.group.WORLD
        n, n2 = ctypes.c_size_t(), ctypes.c_size_t()
        _lib.check(_lib.lib().vgg_ba_reduced_system_doubles(S, model, mode, ctypes.byref(n)), "vgg_ba_reduced_system_doubles")
        _lib.check(_lib.lib().vgg_ba_fabric_doubles(S, model, mode, ctypes.byref(n2)), "vgg_ba_fabric_doubles")
        self.count, self.total = n.value, n2.value
        self.tensor = symm_mem.empty(self.total, dtype=torch.float64, device=device)
        self.handle = symm_mem.rendezvous(self.tensor, group)
        self.tensor.zero_()                           # barrier flags and mailboxes start at zero on every rank
        torch.cuda.synchronize(device)
        dist.barrier(group=group)
        self.multicast_ptr = int(getattr(self.handle, "multicast_ptr", 0) or 0)
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        ptrs = getattr(self.handle, "buffer_ptrs", None)
        self.peer_ptrs = [int(p) for p in ptrs] if ptrs is not None else []
        self.ok = self.multicast_ptr != 0 and len(self.peer_ptrs) == self.world and 1 < self.world <= 8
        self.v2 = self.ok                             # bench.py reads this name

    def struct(self):
        f = _lib.BAFabric()
        f.ar_local, f.ar_multicast, f.ar_doubles = self.tensor.data_ptr(), self.multicast_ptr, self.count
        f.world, f.rank, f.total_doubles = self.world, self.rank, self.total
        for r, p in enumerate(self.peer_ptrs):
            f.peer_base[r] = p
        return f


class AllReduceHook:
    """vgg_allreduce_fn implemented with torch.distributed on views of the solver workspace.  With a usable FabricBuffer
    attached, every reduction of the LM loop is done by the kernels themselves and the solver never calls this hook."""

    def __init__(self, group=None, fabric: "FabricBuffer | None" = None):
        self.group = group
        self.fabric = fabric if (fabric is not None and fabric.ok) else None
        self.calls = 0
        self.bytes = 0
        self.barriers = 0                             # always 0 (the barriers are kernels); bench.py reports it
        self._ws = None
        self._cb = None

    def bind(self, ws: torch.Tensor):
        self._ws = ws
        base = ws.data_ptr()

        def _fn(user, buf, count, op, stream):
            try:
                off = buf - base
                view = self._ws[off:off + count * 8].view(torch.float64)
                dist.all_reduce(view, op=dist.ReduceOp.SUM if op == 0 else dist.ReduceOp.MAX, group=self.group)
                self.calls += 1
                self.bytes += count * 8
                return 0
            except Exception as e:  # surfaces as rc != 0 -> RuntimeError on the Python side
                print(f"[vggsfm_b200.dist] all_reduce failed: {e}", flush=True)
                return -2

        self._cb = _lib.ALLREDUCE_FN(_fn)
        return self._cb


class HostAllReduce:
    """numpy all-reduce with .sum/.max for the oracle's lm_solve (gloo tests of the sharding algebra)."""

    def __init__(self, group=None):
        self.group = group

    def sum(self, arr):
        import numpy as np
        t = torch.from_numpy(np.ascontiguousarray(arr, dtype=np.float64).copy())
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        return t.numpy().reshape(arr.shape)

    def max(self, value):
        t = torch.tensor([float(value)], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
        return float(t[0])
