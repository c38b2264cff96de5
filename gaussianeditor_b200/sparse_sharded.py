"""Sparse exchange for the Gaussian-sharded multi-GPU rasterizer (BASELINE config 4; csrc/sparse_exchange.cu).

Same decomposition as ``sharded.py`` (rank g owns Gaussians ``[g*L, g*L+n_g)`` and tile rows ``ty % world == g``), but a
splat record only travels to the ranks whose tile rows its rectangle touches, and the 2-D gradient sums only travel
back from those ranks: per step and rank the traffic, the depth sort and the gradient reduction shrink from P_total
items to the ~R/V * P_total / world candidates a rank really blends.

  forward   gsr_sparse_preprocess  (preprocess + ordered peer stores of the records into every destination's candidate
                                    array, over NVLink peer mappings)
            gsr_peer_barrier(with_matrix_row)  (flags + count rows through peer memory: the barrier after the push;
                                    every rank learns every segment size -- no NCCL call in the step)
            gsr_sparse_order / gsr_shard_render on the candidates of the owned tile rows
            gsr_frame_broadcast (peer stores of the owned rows into every rank's frame) + barrier
  backward  gsr_shard_backward_render -> gsr_sparse_return (peer stores of the accumulator rows to their owners) + barrier
            gsr_sparse_backward_preprocess (gather in fixed rank order + fused preprocess backward)

The candidate array is in global-index order, so images, depth and the per-tile lists are bit-identical to
``GaussianRasterizer`` on one GPU; gradients agree to summation order.

``SparseRank`` holds the buffers of one rank and the step functions below drive the C ABI for it. With ``peer=None``
several *virtual* ranks can live in one process on one GPU (``link_virtual``): that is how the single-GPU tests cover
everything but the NVLink transport.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import List, Optional

import torch
import torch.nn as nn

from . import _lib
from .rasterizer import GaussianRasterizationSettings, _f32c, _make_cloud, _make_settings, _ptr, _wait_count
from .sharded import ACC_STRIDE, Exchange, PeerWorkspace, ShardPlan, shard_slice

MAXP = 8  # GSR_MAX_PEERS
CTRL_BYTES, CTRL_MATRIX_OFFSET, CTRL_ERROR_OFFSET = 512, 64, 32   # GSR_PEER_CTRL_{BYTES,MATRIX_OFFSET,ERROR_OFFSET}


def _align(n: int, a: int = 256) -> int:
    return (n + a - 1) // a * a


class SparseRank:
    """Buffers of one rank for ONE in-flight forward/backward: local (owner-side) workspace, the peer-visible block
    ``[control words 512 B | frame 4*H*W floats | candidate workspace]`` and small bookkeeping tensors. ``seg_cap`` may
    change from step to step (it only selects how much of the allocated candidate workspace is used); ``cap_alloc`` is
    fixed. ``matrix`` (the [world, 8] segment counts) is a view into the control words: peers write their rows there."""

    def __init__(self, plan: ShardPlan, device, W: int, H: int, cap_alloc: Optional[int] = None,
                 exchange: Optional[Exchange] = None):
        lib = _lib.load()
        self.plan, self.device, self.W, self.H = plan, device, int(W), int(H)
        self.cap_alloc = int(cap_alloc if cap_alloc is not None else max(plan.slice_len, 1))
        self.frame_off = CTRL_BYTES
        self.frame_bytes = CTRL_BYTES + _align(16 * self.W * self.H)   # offset of the candidate workspace in the block
        self.cand_bytes_alloc = lib.gsr_sparse_candidate_bytes(plan.world, self.cap_alloc)
        if self.cand_bytes_alloc == 0:
            _lib.check(-2, "gsr_sparse_candidate_bytes")
        self.total_bytes = self.frame_bytes + self.cand_bytes_alloc
        self.local_bytes = lib.gsr_sparse_local_bytes(max(plan.slice_len, 1))
        with torch.cuda.device(device):
            self.local = torch.empty(self.local_bytes, dtype=torch.uint8, device=device)
            self.radii_local = torch.zeros(max(plan.slice_len, 1), dtype=torch.int32, device=device)
            self.pinned = torch.zeros(2, dtype=torch.int32).pin_memory()
            self.pinned_err = torch.zeros(1, dtype=torch.int32).pin_memory()
            self.peer = None
            if exchange is not None:   # real ranks: CUDA-IPC mapped block, created collectively
                self.peer = PeerWorkspace(self.total_bytes, exchange, device)
                self.block = self.peer.tensor
                self.base_ptrs = list(self.peer.ptrs)
            else:
                self.block = torch.empty(self.total_bytes, dtype=torch.uint8, device=device)
                self.base_ptrs = [None] * plan.world
                self.base_ptrs[plan.rank] = self.block.data_ptr()
            self.block[:CTRL_BYTES].zero_()
            self.matrix = self.block[CTRL_MATRIX_OFFSET:CTRL_MATRIX_OFFSET + 4 * MAXP * MAXP].view(torch.int32).view(MAXP, MAXP)[:plan.world]
            self.err_word = self.block[CTRL_ERROR_OFFSET:CTRL_ERROR_OFFSET + 4].view(torch.int32)
        self.epoch = 0
        if exchange is not None:
            torch.cuda.synchronize(device)
            exchange.barrier(device)      # every rank's control words are zero before anybody raises a flag
            torch.cuda.synchronize(device)
        self.scratch: dict = {}
        self.index = 0
        self._arrays()

    def _arrays(self):
        w = self.plan.world
        self.cand_ptr_array = (C.c_void_p * w)(*[(p + self.frame_bytes) if p is not None else None for p in self.base_ptrs])
        self.frame_ptr_array = (C.c_void_p * w)(*[(p + self.frame_off) if p is not None else None for p in self.base_ptrs])
        self.ctrl_ptr_array = (C.c_void_p * w)(*self.base_ptrs)

    @property
    def cand(self) -> torch.Tensor:
        return self.block[self.frame_bytes:]

    @property
    def frame(self) -> torch.Tensor:
        return self.block[self.frame_off:self.frame_off + 16 * self.W * self.H].view(torch.float32).view(4, self.H, self.W)

    def get(self, name: str, numel: int, dtype, grow: float = 1.0) -> torch.Tensor:
        t = self.scratch.get(name)
        if t is None or t.numel() < numel or t.dtype != dtype:
            t = self.scratch[name] = torch.empty(int(numel * grow) + 256, dtype=dtype, device=self.device)
        return t[:numel]

    def queue_barrier_check(self):
        """Async copy of the control block's sticky error word (set by a peer barrier that timed out) to pinned memory, on
        the current stream; read it with ``raise_if_barrier_failed`` after the next point where the host has waited for
        later work of that stream (the forward does: the instance count arrives behind it)."""
        with torch.cuda.device(self.device):
            self.pinned_err.copy_(self.err_word, non_blocking=True)

    def raise_if_barrier_failed(self):
        if int(self.pinned_err[0]) != 0:
            raise RuntimeError(f"rank {self.plan.rank}: a peer barrier of the sparse exchange timed out (a peer rank died, "
                               "hung or runs a different step sequence); the exchanged data of this step are not valid")

    def close(self):
        self.scratch.clear()
        self.matrix = self.err_word = None
        if self.peer is not None:
            self.block = None
            self.peer.close()
            self.peer = None


def link_virtual(ranks: List[SparseRank]):
    """Virtual ranks in one process: everybody's 'peer mapping' of rank r is simply r's own buffer."""
    ptrs = [r.block.data_ptr() for r in ranks]
    for r in ranks:
        r.base_ptrs = list(ptrs)
        r._arrays()


class SparseStep:
    """One forward in flight on one rank."""
    __slots__ = ("rk", "cap", "s", "keep", "inputs", "M", "R", "max_count", "binning", "img", "radii_cand", "cplan", "n",
                 "__weakref__")


def _cplan(plan: ShardPlan, cap: int) -> "_lib.SparsePlan":
    return _lib.SparsePlan(plan.world, plan.rank, max(plan.slice_len, 1), int(cap))


def sparse_preprocess(rk: SparseRank, rs: GaussianRasterizationSettings, means3D, sh, colors_precomp, opacities, scales,
                      rotations, cov3Ds_precomp, cap: int) -> SparseStep:
    """Owner side: preprocess the shard and push every record to the candidate arrays of the ranks it touches. Writes
    row `rank` of ``rk.matrix`` (the other rows must be zero before the all-reduce that follows)."""
    lib = _lib.load()
    plan, device = rk.plan, rk.device
    if not means3D.is_cuda:
        raise RuntimeError("the rasterizer needs CUDA tensors (there is no CPU path)")
    if means3D.size(0) != plan.count:
        raise RuntimeError(f"rank {plan.rank} owns {plan.count} Gaussians, got {means3D.size(0)}")
    if not (1 <= cap <= rk.cap_alloc):
        raise RuntimeError(f"segment capacity {cap} outside [1, {rk.cap_alloc}]")
    st = SparseStep()
    st.rk, st.cap, st.n = rk, int(cap), plan.count
    st.M = sh.size(1) if sh.numel() != 0 else 0
    with torch.cuda.device(device):
        means3D = _f32c(means3D, device); opacities = _f32c(opacities, device)
        sh = _f32c(sh, device); colors_precomp = _f32c(colors_precomp, device)
        scales = _f32c(scales, device); rotations = _f32c(rotations, device)
        cov3Ds_precomp = _f32c(cov3Ds_precomp, device)
        st.inputs = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
        st.keep = []
        st.s = _make_settings(rs, st.M, device, st.keep)
        st.cplan = _cplan(plan, cap)
        c = _make_cloud(plan.count, *[st.inputs[i] for i in (0, 3, 1, 2, 4, 5, 6)])
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        # (the count matrix is never zeroed: every step each rank rewrites its whole row, here and -- through
        # peer_barrier(with_row=True) -- in every peer's copy; a zero-fill could wipe a faster peer's fresh row)
        cand_bytes = lib.gsr_sparse_candidate_bytes(plan.world, cap)
        _lib.check(lib.gsr_sparse_preprocess(C.byref(st.s), C.byref(c), C.byref(st.cplan), _ptr(rk.local), rk.local_bytes,
                                             _ptr(rk.radii_local), rk.cand_ptr_array, cand_bytes,
                                             C.c_void_p(rk.matrix[plan.rank].data_ptr()), stream),
                   "gsr_sparse_preprocess")
    return st


def sparse_order(st: SparseStep):
    """Tile-owner side, after the count matrix is complete and every push has landed: candidates -> depth order + scan.
    Returns (num_rendered of this rank, largest segment count anywhere); one stream synchronisation."""
    lib = _lib.load()
    rk = st.rk
    with torch.cuda.device(rk.device):
        M = rk.plan.world * st.cap
        st.radii_cand = rk.get("radii_cand", M, torch.int32, grow=1.25)
        stream = torch.cuda.current_stream(rk.device)
        cand_bytes = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
        rk.pinned[0] = -1   # both words are copied out BEFORE the depth sort is queued: the host gets them early
        _lib.check(lib.gsr_sparse_order(C.byref(st.s), C.byref(st.cplan), _ptr(rk.cand), cand_bytes, _ptr(rk.matrix),
                                        _ptr(st.radii_cand), C.c_void_p(rk.pinned.data_ptr()),
                                        C.c_void_p(stream.cuda_stream)), "gsr_sparse_order")
        st.R = _wait_count(rk.pinned, stream.synchronize)   # the max-count word was copied just before it
        st.max_count = int(rk.pinned[1])
    return st.R, st.max_count


def sparse_render(st: SparseStep, color: torch.Tensor, depth: torch.Tensor):
    """Bin + blend the owned tiles of the candidate cloud into `color` [3,H,W] / `depth` [1,H,W] (other rows untouched)."""
    lib = _lib.load()
    rk = st.rk
    with torch.cuda.device(rk.device):
        M, R, W, H = rk.plan.world * st.cap, st.R, rk.W, rk.H
        bbytes = lib.gsr_binning_bytes(M, R, W, H) if R > 0 else 0
        st.binning = rk.get("binning", bbytes, torch.uint8, grow=1.25)
        ibytes = lib.gsr_image_bytes(W, H)
        st.img = rk.get("img", ibytes, torch.uint8)
        own = rk.plan.owner()
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        gb = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
        _lib.check(lib.gsr_shard_render(C.byref(st.s), C.byref(own), M, R, _ptr(rk.cand), gb, _ptr(st.binning), bbytes,
                                        _ptr(st.img), ibytes, _ptr(st.radii_cand), _ptr(color), _ptr(depth), stream),
                   "gsr_shard_render")


def frame_broadcast(rk: SparseRank):
    """Peer stores of this rank's owned rows of ``rk.frame`` into every other rank's frame (barrier must follow)."""
    lib = _lib.load()
    with torch.cuda.device(rk.device):
        own = rk.plan.owner()
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        _lib.check(lib.gsr_frame_broadcast(C.byref(own), rk.W, rk.H, _ptr(rk.frame), rk.frame_ptr_array, stream),
                   "gsr_frame_broadcast")


def peer_barrier(rk: SparseRank, with_row: bool = False):
    """Cross-rank barrier on the compute stream through the control words of the peer-mapped blocks (gsr_peer_barrier):
    work queued behind it starts once every rank has reached the same point; with `with_row` this rank's row of the
    count matrix is first copied into every peer's matrix (the all-gather of the segment sizes)."""
    lib = _lib.load()
    rk.epoch += 1
    with torch.cuda.device(rk.device):
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        _lib.check(lib.gsr_peer_barrier(rk.plan.world, rk.plan.rank, rk.ctrl_ptr_array, rk.epoch & 0xFFFFFFFF,
                                        1 if with_row else 0, stream), "gsr_peer_barrier")


def sparse_backward_render(st: SparseStep, grad_out_color: torch.Tensor) -> torch.Tensor:
    lib = _lib.load()
    rk = st.rk
    with torch.cuda.device(rk.device):
        M = rk.plan.world * st.cap
        grad_out_color = _f32c(grad_out_color, rk.device)
        acc = rk.get("acc", M * ACC_STRIDE, torch.float32, grow=1.25).view(M, ACC_STRIDE)
        own = rk.plan.owner()
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        gb = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
        _lib.check(lib.gsr_shard_backward_render(C.byref(st.s), C.byref(own), M, st.R, _ptr(rk.cand), gb, _ptr(st.binning),
                                                 st.binning.numel(), _ptr(st.img), st.img.numel(), _ptr(grad_out_color),
                                                 _ptr(acc), acc.numel() * 4, stream), "gsr_shard_backward_render")
    return acc


def sparse_return(st: SparseStep, acc: torch.Tensor):
    """Peer stores of every candidate's accumulator row into its owner's `ret` array (barrier must follow)."""
    lib = _lib.load()
    rk = st.rk
    with torch.cuda.device(rk.device):
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        _lib.check(lib.gsr_sparse_return(C.byref(st.cplan), _ptr(acc), _ptr(rk.matrix), rk.cand_ptr_array, stream),
                   "gsr_sparse_return")


def sparse_backward_preprocess(st: SparseStep):
    """Owner side: add the returned rows of every Gaussian (ascending rank) and run the fused preprocess backward."""
    lib = _lib.load()
    rk = st.rk
    device, n, M = rk.device, st.n, st.M
    (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp) = st.inputs
    with torch.cuda.device(device):
        f32 = dict(dtype=torch.float32, device=device)
        dL_dmeans3D = torch.empty(n, 3, **f32); dL_dmeans2D = torch.empty(n, 3, **f32)
        dL_dcolors = torch.empty(n, 3, **f32); dL_dopacity = torch.empty(n, 1, **f32)
        dL_dcov3D = torch.empty(n, 6, **f32); dL_dsh = torch.empty(n, M, 3, **f32)
        dL_dscales = torch.empty(n, 3, **f32); dL_drotations = torch.empty(n, 4, **f32)
        if n > 0:
            c = _make_cloud(n, means3D, opacities, sh, colors_precomp, scales, rotations, cov3Ds_precomp)
            gr = _lib.Grads(_ptr(dL_dmeans3D), _ptr(dL_dmeans2D), _ptr(dL_dcolors), _ptr(dL_dopacity),
                            _ptr(dL_dcov3D), _ptr(dL_dsh), _ptr(dL_dscales), _ptr(dL_drotations))
            acc_slice = rk.get("acc_slice", n * ACC_STRIDE, torch.float32)
            stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
            gb = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
            _lib.check(lib.gsr_sparse_backward_preprocess(C.byref(st.s), C.byref(c), C.byref(st.cplan), _ptr(rk.local),
                                                          rk.local_bytes, _ptr(rk.radii_local), _ptr(rk.cand), gb,
                                                          _ptr(acc_slice), acc_slice.numel() * 4, C.byref(gr), stream),
                       "gsr_sparse_backward_preprocess")
            if scales.numel() == 0:
                dL_dscales.zero_(); dL_drotations.zero_()
    return (dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D)


def next_capacity(max_count: int, cap_alloc: int) -> int:
    """Segment capacity for the next step from the largest segment seen (identical on every rank: the count matrix is
    all-reduced): 10 % headroom (every slot of headroom is a hole the depth sort still carries), 4096-slot granularity,
    never above what was allocated. A frame that overflows is simply redone with the exact requirement."""
    want = int(max_count * 1.10) + 4096
    return max(1, min(cap_alloc, (want + 4095) // 4096 * 4096))


# ---------------------------------------------------------------------------------------------------------
# autograd + pool (one process per GPU)
# ---------------------------------------------------------------------------------------------------------
class SparsePool:
    """`depth` SparseRanks created COLLECTIVELY up front (peer allocation is a collective: creating them lazily inside a
    forward would hang as soon as the ranks disagree on the number of live forwards). A rank is taken per forward and
    given back when that forward's state dies; every rank runs the same sequence, so workspace k here is always paired
    with workspace k on the peers. Also holds the adaptive segment capacity shared by all ranks."""

    def __init__(self, plan: ShardPlan, device, W, H, exchange: Exchange, depth: int = 2):
        self.all = []
        for k in range(depth):
            rk = SparseRank(plan, device, W, H, exchange=exchange)
            rk.index = k
            self.all.append(rk)
        self.free = list(self.all)
        self.cap = self.all[0].cap_alloc     # first step: worst case; adapts after the first count matrix
        self.redo = 0                        # forwards that had to be repeated because a segment overflowed

    def take(self) -> SparseRank:
        if not self.free:
            raise RuntimeError(f"more than {len(self.all)} sharded forwards alive at once: construct "
                               f"ShardedGaussianRasterizer(..., max_in_flight=N) with a larger N")
        return self.free.pop(0)

    def give(self, rk: SparseRank):
        self.free.append(rk)
        self.free.sort(key=lambda r: r.index)

    def close(self):
        for rk in self.all:
            rk.close()
        self.all, self.free = [], []


TRACE = None   # set to a list to collect (phase name, CUDA event) marks of the autograd path (bench.py, diagnostics)


def _mark(name: str):
    if TRACE is not None:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        TRACE.append((name, ev))


class _SparseShardedRasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, pool, exchange):
        rk = pool.take()
        device = means3D.device
        _mark("start")
        try:
            while True:
                st = sparse_preprocess(rk, rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                       pool.cap)
                _mark("preprocess+push")
                peer_barrier(rk, with_row=True)                # counts + barrier: every push has landed
                rk.queue_barrier_check()                       # sticky error word (this and earlier barriers) -> pinned
                _mark("count all-reduce")
                R, max_count = sparse_order(st)                # waits for R, queued behind that copy
                rk.raise_if_barrier_failed()
                _mark("order")
                if max_count <= st.cap:
                    break
                pool.redo += 1                                  # same decision on every rank (the matrix is global)
                pool.cap = next_capacity(max_count, rk.cap_alloc)
        except BaseException:
            pool.give(rk)                                       # a failed forward must not leak its workspace
            raise
        pool.cap = next_capacity(max_count, rk.cap_alloc)
        weakref.finalize(st, pool.give, rk)
        # Every pixel has exactly one writer (the owner of its tile row; empty tiles are written too), so the frame needs
        # no zero-fill -- and must not get one: a faster peer may already have stored its rows here.
        frame = rk.frame
        sparse_render(st, frame[:3], frame[3:])
        _mark("bin+blend")
        frame_broadcast(rk)
        peer_barrier(rk)
        out = frame.clone()                                 # the peer-visible frame is overwritten by the next step
        _mark("frame broadcast+barrier")
        ctx.st, ctx.exchange = st, exchange
        radii = rk.radii_local[:rk.plan.count].clone()
        ctx.mark_non_differentiable(radii)
        _SparseShardedRasterize.last = dict(R=R, cap=st.cap, max_count=max_count)
        return out[:3], radii, out[3:]

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth):
        st, exchange = ctx.st, ctx.exchange
        if st is None:
            raise RuntimeError("the sharded rasterizer's backward can run once (its workspace went back to the pool)")
        _mark("loss")
        acc = sparse_backward_render(st, grad_out_color)
        _mark("blend backward")
        sparse_return(st, acc)
        peer_barrier(st.rk)
        _mark("return push+barrier")
        grads = sparse_backward_preprocess(st)
        _mark("gather+preprocess backward")
        ctx.st = None   # the workspace goes back to the pool now, not when the output tensors die
        return (*grads, None, None, None)
