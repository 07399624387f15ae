"""Multi-GPU plumbing for the rasterizer path: views shard one per GPU, ONE all-reduce per step.

The reference is single-process / single-GPU (src/utils/general_utils.py:143 pins cuda:0; no
collective call sites anywhere, SURVEY.md section 2.2), so this is new functionality whose parity
gate is  allreduce(grads) == sum over ranks of the single-GPU gradient of that rank's view.

A training step consumes one camera (src/train_gaussians.py:103-110) and cameras are independent
given the same Gaussians, so the path shards by view with no collective inside the op.  The only
exchange is the sum of the per-Gaussian gradients, which the backward already writes into one flat
float32 arena (`_C.rasterize_gaussians_backward_arena`): the arena IS the NCCL buffer, no packing
copy.  torch.distributed (NCCL over NVLink/NVSwitch, gloo in CPU tests) is plumbing.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist


def views_for_step(step: int, rank: int, world_size: int, num_cameras: int) -> int:
    """Camera index rendered by `rank` at optimiser step `step`: consecutive blocks of `world_size`
    cameras per step, wrapping around the camera list (one view per GPU per step)."""
    if not (0 <= rank < world_size):
        raise ValueError("rank out of range")
    return (step * world_size + rank) % num_cameras


def epoch_schedule(world_size: int, num_cameras: int) -> List[List[int]]:
    """All steps of one pass over the cameras: ceil(num_cameras / world_size) steps, each a list of
    `world_size` camera ids (the last step wraps)."""
    steps = (num_cameras + world_size - 1) // world_size
    return [[views_for_step(s, r, world_size, num_cameras) for r in range(world_size)] for s in range(steps)]


def trainable_slice(flat: torch.Tensor, num_gaussians: int, call_shape: str = "native") -> torch.Tensor:
    """The contiguous prefix of the gradient arena that the optimizer consumes.

    `native` (the op computes covariances from scales/rotations): rotations, colors, opacity,
    means3D, scales = the first 21 floats per Gaussian (each segment padded to a multiple of 4 floats,
    `_C.trainable_floats`); means2D (densification statistics only) and the conic / cov3D segments behind
    it need not travel.  Any other call shape: the whole arena.
    """
    from . import _C
    if call_shape == "native":
        return flat[: _C.trainable_floats(num_gaussians)]
    return flat


def allreduce_gradient_arena(flat: torch.Tensor, group: Optional[dist.ProcessGroup] = None,
                             average: bool = False, async_op: bool = False):
    """Sum (or mean) the flat gradient arena (or a `trainable_slice` of it) over all ranks with a
    single collective.

    No-op when torch.distributed is not initialised or the world has one rank.  With
    `async_op=True` returns the work handle so the caller can overlap the next view's forward.
    """
    if not dist.is_available() or not dist.is_initialized():
        return None
    world = dist.get_world_size(group)
    if world == 1:
        return None
    work = dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
    if average:
        if async_op:
            work.wait()
        flat.div_(world)
        return None
    return work


def allreduce_densification_stats(grad_accum: torch.Tensor, denom: torch.Tensor, max_radii2D: torch.Tensor,
                                  group: Optional[dist.ProcessGroup] = None) -> None:
    """Keep the densification statistics replica-consistent (src/train_gaussians.py:161-164,
    src/scene/gaussian_model.py:739-741): SUM for the accumulated view-space gradient norm and its
    denominator, MAX for the largest screen radius."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    dist.all_reduce(grad_accum, op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(denom, op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(max_radii2D, op=dist.ReduceOp.MAX, group=group)


class PeerAllReduce:
    """Sum a float32 gradient arena over the GPUs of one node with `gh_allreduce_p2p`: one kernel per
    rank that reads and writes the peers' arenas through NVLink (symmetric memory), instead of NCCL.

        par = PeerAllReduce(_C.arena_floats(P), device)          # once; collective (rendezvous)
        flat, grads, _ = _C.rasterize_gaussians_backward_arena(..., arena_storage=par.buffer)
        par.all_reduce(n_floats=_C.trainable_floats(P))          # in place, on the current stream
        optimizer.step(..., skip_flags=(par.error_flag,), nan_flag_in=par.nan_flag)   # stream order is enough

    `use_multicast`: None = choose by world size (NVLS multimem from 8 GPUs up, when the allocation has a
    multicast mapping), True / False = force.  Every rank must call `all_reduce` the same number of times
    with the same range.  A peer that does not arrive within GH_ALLREDUCE_TIMEOUT_MS (default 30 s) makes the
    kernel SKIP the reduction and raise `error_flag` (device uint32, sticky); hand it to the optimizer as a
    skip flag (no host sync) or poll `ok()` (host sync; `all_reduce(check=True)` raises).  `nan_flag`
    (device uint32, identical on all ranks) tells whether the reduced range holds a NaN: the optimizer's NaN
    guard without its own pass over the gradients."""

    def __init__(self, numel: int, device: torch.device, group: Optional[dist.ProcessGroup] = None,
                 use_multicast: Optional[bool] = None):
        import ctypes as C
        import torch.distributed._symmetric_memory as symm_mem
        from . import _capi
        if not dist.is_initialized():
            raise RuntimeError("PeerAllReduce needs an initialised torch.distributed process group")
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        if self.world > 16:
            raise RuntimeError("PeerAllReduce supports up to 16 GPUs of one node")
        self.device = device
        n = (int(numel) + 3) // 4 * 4
        with torch.cuda.device(device):
            self.buffer = symm_mem.empty(n, dtype=torch.float32, device=device)
            self._flags = symm_mem.empty(64, dtype=torch.int32, device=device)
            self._flags.zero_()
            self.buffer.zero_()                                     # segment padding never holds garbage
            self._local = torch.zeros(8, dtype=torch.int32, device=device)
            self.nan_flag = torch.zeros(1, dtype=torch.int32, device=device)
            hb = symm_mem.rendezvous(self.buffer, self.group)
            hf = symm_mem.rendezvous(self._flags, self.group)
            torch.cuda.synchronize(device)
        dist.barrier(self.group)                                   # every rank's flag block is zero before anyone signals
        self._handles = (hb, hf)                                   # keep the mappings alive
        self._bufs = (C.c_ulonglong * self.world)(*[int(p) for p in hb.buffer_ptrs])
        self._flagptrs = (C.c_ulonglong * self.world)(*[int(p) for p in hf.buffer_ptrs])
        mc = int(getattr(hb, "multicast_ptr", 0) or 0)
        if use_multicast is None:
            # measured (tools/allreduce_case.py, 42 MB): peer loads/stores win up to 4 GPUs (85 us at 2), NVLS multimem at 8
            # (121 us against 157 us peer and 195 us NCCL)
            use_multicast = self.world >= 8
        self.multicast = mc if use_multicast else 0
        self._epoch = 0
        self._lib = _capi.load()
        self._capi = _capi

    @property
    def error_flag(self) -> torch.Tensor:
        """Device uint32 (view): non-zero once any all-reduce of this object failed (peer timeout)."""
        return self._local[2:3]

    def all_reduce(self, n_floats: Optional[int] = None, offset_floats: int = 0, check: bool = False) -> None:
        import ctypes as C
        n = self.buffer.numel() - offset_floats if n_floats is None else int(n_floats)
        n = (n + 3) // 4 * 4
        if offset_floats % 4 or offset_floats + n > self.buffer.numel():
            raise RuntimeError("PeerAllReduce: range must be 4-float aligned and inside the buffer")
        self._epoch += 1
        with torch.cuda.device(self.device):
            self._capi.check(self._lib.gh_allreduce_p2p(
                self._bufs, self._flagptrs, C.c_ulonglong(self.multicast), self.rank, self.world,
                C.c_size_t(offset_floats), C.c_size_t(n), C.c_uint(self._epoch),
                self._capi._ptr(self._local), self._capi._ptr(self.nan_flag), self._capi._stream(self.device)))
        if check and not self.ok():
            raise RuntimeError("PeerAllReduce: a peer did not reach the barrier in time; the reduction was skipped "
                               "and the gradient arena is undefined (GH_ALLREDUCE_TIMEOUT_MS)")

    def ok(self) -> bool:
        return int(self._local[2].item()) == 0
