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
from .rasterizer import GaussianRasterizationSettings, _f32c, _make_settings, _ptr, _wait_count
from .sharded import (ACC_STRIDE, Exchange, PeerWorkspace, ShardPlan, _shard_cloud, grads_in_slots, mask_ptr,
                      preprocess_grads, shard_slice)

MAXP = 8  # GSR_MAX_PEERS
CTRL_BYTES, CTRL_MATRIX_OFFSET, CTRL_ERROR_OFFSET = 512, 64, 32   # GSR_PEER_CTRL_{BYTES,MATRIX_OFFSET,ERROR_OFFSET}
CTRL_EPOCH_OFFSET, CTRL_STATUS_OFFSET = 320, 352   # GSR_PEER_CTRL_{EPOCH,STATUS}_OFFSET (device-epoch barrier)
AW_CNT_SLOT = 11   # GSR_SPARSE_AW_CNT_SLOT: float of an apply_weights candidate row that carries the int32 count bits
ROW_FLOATS = 64    # GSR_PEER_ROW_FLOATS: floats per slot of gsr_peer_row_put
CAM_SLOT_BYTES = 4 * MAXP * ROW_FLOATS   # the camera-gradient slots of a block (only with camera_grad)


def _align(n: int, a: int = 256) -> int:
    return (n + a - 1) // a * a


class SparseRank:
    """Buffers of one rank for ONE in-flight forward/backward: local (owner-side) workspace, the peer-visible block
    ``[control words 512 B | frame 4*H*W floats | candidate workspace]`` and small bookkeeping tensors. ``seg_cap`` may
    change from step to step (it only selects how much of the allocated candidate workspace is used); ``cap_alloc`` is
    fixed. ``matrix`` (the [world, 8] segment counts) is a view into the control words: peers write their rows there.
    ``alpha``: the frame has a fifth plane (the alpha image). ``camera``: the camera-gradient slots
    [GSR_MAX_PEERS, GSR_PEER_ROW_FLOATS] floats follow the frame (slot r is written by rank r, gsr_peer_row_put)."""

    def __init__(self, plan: ShardPlan, device, W: int, H: int, cap_alloc: Optional[int] = None,
                 exchange: Optional[Exchange] = None, alpha: bool = False, camera: bool = False):
        lib = _lib.load()
        self.plan, self.device, self.W, self.H = plan, device, int(W), int(H)
        self.cap_alloc = int(cap_alloc if cap_alloc is not None else max(plan.slice_len, 1))
        self.planes = 5 if alpha else 4
        self.frame_off = CTRL_BYTES
        self.cam_off = CTRL_BYTES + _align(4 * self.planes * self.W * self.H)
        # offset of the candidate workspace in the block
        self.frame_bytes = self.cam_off + (CAM_SLOT_BYTES if camera else 0)
        self.camera = bool(camera)
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
            # device-epoch barrier: this rank's barrier counter and the overflow words the ranks sent with their barriers
            self.epoch_word = self.block[CTRL_EPOCH_OFFSET:CTRL_EPOCH_OFFSET + 4].view(torch.int32)
            self.status_array = self.block[CTRL_STATUS_OFFSET:CTRL_STATUS_OFFSET + 4 * MAXP].view(torch.int32)[:plan.world]
        self.epoch = 0
        self.device_epoch = False   # True: every barrier on this block is gsr_peer_barrier_device (static forward)
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
        self.cam_ptr_array = (C.c_void_p * w)(*[(p + self.cam_off) if p is not None else None for p in self.base_ptrs])

    @property
    def cand(self) -> torch.Tensor:
        return self.block[self.frame_bytes:]

    @property
    def frame(self) -> torch.Tensor:
        n = self.planes * self.W * self.H
        return self.block[self.frame_off:self.frame_off + 4 * n].view(torch.float32).view(self.planes, self.H, self.W)

    @property
    def cam_slots(self) -> torch.Tensor:
        """[world, ROW_FLOATS] float32: slot r holds rank r's camera partial after the barrier that follows the puts."""
        if not self.camera:
            raise RuntimeError("this SparseRank was built without camera slots")
        v = self.block[self.cam_off:self.cam_off + CAM_SLOT_BYTES].view(torch.float32).view(MAXP, ROW_FLOATS)
        return v[:self.plan.world]

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
        self.matrix = self.err_word = self.epoch_word = self.status_array = None
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
                 "grad_mask", "__weakref__")


def _cplan(plan: ShardPlan, cap: int) -> "_lib.SparsePlan":
    return _lib.SparsePlan(plan.world, plan.rank, max(plan.slice_len, 1), int(cap))


def sparse_preprocess(rk: SparseRank, rs: GaussianRasterizationSettings, means3D, sh, colors_precomp, opacities, scales,
                      rotations, cov3Ds_precomp, cap: int, raw_rest: Optional[torch.Tensor] = None,
                      grad_mask: Optional[torch.Tensor] = None) -> SparseStep:
    """Owner side: preprocess the shard and push every record to the candidate arrays of the ranks it touches. Writes
    row `rank` of ``rk.matrix`` (the other rows must be zero before the all-reduce that follows). `raw_rest`: a raw
    shard, `grad_mask`: this rank's edit mask [n] (the records carry the edit words), as in sharded.shard_preprocess."""
    lib = _lib.load()
    plan, device = rk.plan, rk.device
    if not means3D.is_cuda:
        raise RuntimeError("the rasterizer needs CUDA tensors (there is no CPU path)")
    if means3D.size(0) != plan.count:
        raise RuntimeError(f"rank {plan.rank} owns {plan.count} Gaussians, got {means3D.size(0)}")
    if not (1 <= cap <= rk.cap_alloc):
        raise RuntimeError(f"segment capacity {cap} outside [1, {rk.cap_alloc}]")
    st = SparseStep()
    st.rk, st.cap, st.n, st.grad_mask = rk, int(cap), plan.count, grad_mask
    st.M = sh.size(1) if sh.numel() != 0 else 0
    if raw_rest is not None:
        st.M = 1 + raw_rest.size(1)
    with torch.cuda.device(device):
        means3D = _f32c(means3D, device); opacities = _f32c(opacities, device)
        sh = _f32c(sh, device); colors_precomp = _f32c(colors_precomp, device)
        scales = _f32c(scales, device); rotations = _f32c(rotations, device)
        cov3Ds_precomp = _f32c(cov3Ds_precomp, device)
        st.inputs = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
        if raw_rest is not None:   # a slice whose rows start off a 16-byte boundary is cloned by _f32c
            st.inputs = st.inputs + (_f32c(raw_rest, device),)
        raw = ("_raw" if raw_rest is not None else "") + ("_masked" if grad_mask is not None else "")
        masked = () if grad_mask is None else (mask_ptr(grad_mask),)
        st.keep = []
        st.s = _make_settings(rs, st.M, device, st.keep)
        st.cplan = _cplan(plan, cap)
        c = _shard_cloud(plan.count, st.inputs)
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        # (the count matrix is never zeroed: every step each rank rewrites its whole row, here and -- through
        # peer_barrier(with_row=True) -- in every peer's copy; a zero-fill could wipe a faster peer's fresh row)
        cand_bytes = lib.gsr_sparse_candidate_bytes(plan.world, cap)
        _lib.check(getattr(lib, "gsr_sparse_preprocess" + raw)(
            C.byref(st.s), C.byref(c), C.byref(st.cplan), _ptr(rk.local), rk.local_bytes, _ptr(rk.radii_local),
            rk.cand_ptr_array, cand_bytes, C.c_void_p(rk.matrix[plan.rank].data_ptr()), *masked, stream),
            "gsr_sparse_preprocess" + raw)
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


def sparse_alpha(st: SparseStep, alpha: torch.Tensor):
    """After sparse_render: alpha = 1 - final_T on the owned tile rows of `alpha` [1,H,W] (other rows untouched)."""
    lib = _lib.load()
    rk = st.rk
    with torch.cuda.device(rk.device):
        own = rk.plan.owner()
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        _lib.check(lib.gsr_shard_alpha_image(C.byref(own), _ptr(st.img), st.img.numel(), rk.W, rk.H, _ptr(alpha),
                                             stream), "gsr_shard_alpha_image")


def frame_broadcast(rk: SparseRank):
    """Peer stores of this rank's owned rows of ``rk.frame`` (all its planes) into every other rank's frame (barrier
    must follow)."""
    lib = _lib.load()
    with torch.cuda.device(rk.device):
        own = rk.plan.owner()
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        if rk.planes == 4:
            _lib.check(lib.gsr_frame_broadcast(C.byref(own), rk.W, rk.H, _ptr(rk.frame), rk.frame_ptr_array, stream),
                       "gsr_frame_broadcast")
        else:
            _lib.check(lib.gsr_frame_broadcast_planes(C.byref(own), rk.W, rk.H, rk.planes, _ptr(rk.frame),
                                                      rk.frame_ptr_array, stream), "gsr_frame_broadcast_planes")


def camera_put(rk: SparseRank, row: torch.Tensor):
    """Peer stores of this rank's camera partial `row` [CAM_ROW] into slot `rank` of every rank's camera slots
    (gsr_peer_row_put). A peer_barrier must follow, and the slots must be read (combine_camera_rows on
    ``rk.cam_slots``) before this rank's next barrier on the block."""
    from .sharded import CAM_ROW
    lib = _lib.load()
    with torch.cuda.device(rk.device):
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        _lib.check(lib.gsr_peer_row_put(rk.plan.world, rk.plan.rank, _ptr(row), CAM_ROW, rk.cam_ptr_array, stream),
                   "gsr_peer_row_put")


def peer_barrier(rk: SparseRank, with_row: bool = False, status_word: Optional[torch.Tensor] = None):
    """Cross-rank barrier on the compute stream through the control words of the peer-mapped blocks (gsr_peer_barrier):
    work queued behind it starts once every rank has reached the same point; with `with_row` this rank's row of the
    count matrix is first copied into every peer's matrix (the all-gather of the segment sizes). On a block of a static
    module (``rk.device_epoch``) it is gsr_peer_barrier_device, which can be replayed in a CUDA graph; `status_word`
    (device int32 [1]) then lands in slot `rank` of every rank's ``status_array``."""
    lib = _lib.load()
    if rk.device_epoch:
        with torch.cuda.device(rk.device):
            stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
            _lib.check(lib.gsr_peer_barrier_device(rk.plan.world, rk.plan.rank, rk.ctrl_ptr_array, 1 if with_row else 0,
                                                   _ptr(status_word), stream), "gsr_peer_barrier_device")
        return
    if status_word is not None:
        raise RuntimeError("a status word travels with device-epoch barriers only")
    rk.epoch += 1
    with torch.cuda.device(rk.device):
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        _lib.check(lib.gsr_peer_barrier(rk.plan.world, rk.plan.rank, rk.ctrl_ptr_array, rk.epoch & 0xFFFFFFFF,
                                        1 if with_row else 0, stream), "gsr_peer_barrier")


def sparse_backward_render(st: SparseStep, grad_out_color: torch.Tensor, deterministic: bool = False,
                           grad_depth: Optional[torch.Tensor] = None,
                           grad_alpha: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Blend backward of the owned tiles into the candidate accumulators [world*cap, 12] (deterministic: no float
    atomics, every row written; `grad_depth`: dL/dz in float 9 too; `grad_alpha`: the alpha image's gradient too)."""
    from .sharded import owner_backward_render
    lib = _lib.load()
    rk = st.rk
    M = rk.plan.world * st.cap
    acc = rk.get("acc", M * ACC_STRIDE, torch.float32, grow=1.25).view(M, ACC_STRIDE)
    gb = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
    owner_backward_render(st.s, rk.plan.owner(), M, st.R, rk.cand[:gb], st.binning, st.img, grad_out_color, acc,
                          deterministic, lambda name, n, dtype, grow: rk.get(name, n, dtype, grow), grad_depth,
                          grad_alpha, st.grad_mask is not None)
    return acc


def sparse_return(st: SparseStep, acc: torch.Tensor):
    """Peer stores of every candidate's accumulator row into its owner's `ret` array (barrier must follow)."""
    lib = _lib.load()
    rk = st.rk
    with torch.cuda.device(rk.device):
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        _lib.check(lib.gsr_sparse_return(C.byref(st.cplan), _ptr(acc), _ptr(rk.matrix), rk.cand_ptr_array, stream),
                   "gsr_sparse_return")


def sparse_backward_preprocess(st: SparseStep, depth: bool = False, camera: Optional[_lib.CameraGrads] = None):
    """Owner side: add the returned rows of every Gaussian (ascending rank) and run the fused preprocess backward
    (`depth`: the rows carry dL/dz). Gradients in the order of sharded.shard_backward_preprocess. `camera` (from
    sharded.camera_row): this rank's camera partial is written too (gsr_sparse_backward_preprocess_camera)."""
    lib = _lib.load()
    rk = st.rk
    n = st.n

    def call(c, gr, raw):
        acc_slice = rk.get("acc_slice", n * ACC_STRIDE, torch.float32)
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        gb = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
        args = (C.byref(st.s), C.byref(c), C.byref(st.cplan), _ptr(rk.local), rk.local_bytes, _ptr(rk.radii_local),
                _ptr(rk.cand), gb, _ptr(acc_slice), acc_slice.numel() * 4, C.byref(gr))
        if st.grad_mask is not None:
            if raw:
                _lib.check(lib.gsr_sparse_backward_preprocess_raw_masked(*args, int(depth), mask_ptr(st.grad_mask),
                                                                         stream), "gsr_sparse_backward_preprocess_raw_masked")
            else:
                _lib.check(lib.gsr_sparse_backward_preprocess_masked(*args, int(depth), None, mask_ptr(st.grad_mask),
                                                                     stream), "gsr_sparse_backward_preprocess_masked")
        elif camera is not None:
            _lib.check(lib.gsr_sparse_backward_preprocess_camera(*args, int(depth), C.byref(camera), stream),
                       "gsr_sparse_backward_preprocess_camera")
        elif raw:
            _lib.check(lib.gsr_sparse_backward_preprocess_raw(*args, int(depth), stream),
                       "gsr_sparse_backward_preprocess_raw")
        elif depth:
            _lib.check(lib.gsr_sparse_backward_preprocess_depth(*args, stream), "gsr_sparse_backward_preprocess_depth")
        else:
            _lib.check(lib.gsr_sparse_backward_preprocess(*args, stream), "gsr_sparse_backward_preprocess")
    return preprocess_grads(lib, n, st.M, st.inputs, rk.device, call)


def sparse_order_static(st: SparseStep, capacity: int):
    """sparse_order without the host words (gsr_sparse_order_static): R and the largest segment stay on the device (the
    status kernel of sparse_render_static reads them), and ``st.R = capacity`` sizes the binning and the backward."""
    lib = _lib.load()
    rk = st.rk
    with torch.cuda.device(rk.device):
        M = rk.plan.world * st.cap
        st.radii_cand = rk.get("radii_cand", M, torch.int32)
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        cand_bytes = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
        _lib.check(lib.gsr_sparse_order_static(C.byref(st.s), C.byref(st.cplan), _ptr(rk.cand), cand_bytes,
                                               _ptr(rk.matrix), _ptr(st.radii_cand), stream), "gsr_sparse_order_static")
    st.R = int(capacity)
    st.max_count = None


def sparse_render_static(st: SparseStep, color: torch.Tensor, depth: torch.Tensor, status: torch.Tensor):
    """sparse_render for the capacity of sparse_order_static (gsr_shard_render_static with the count matrix): status
    gets {R, R > capacity or a segment > seg_cap, largest segment, 0} and the owned tiles are emptied on overflow."""
    from .sharded import render_static
    lib = _lib.load()
    rk = st.rk
    M = rk.plan.world * st.cap
    gb = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
    st.binning, st.img = render_static(st.s, rk.plan.owner(), M, st.R, rk.cand[:gb], st.radii_cand, color, depth,
                                       status, lambda name, n, dtype, grow: rk.get(name, n, dtype, grow), rk.matrix,
                                       rk.plan.world, st.cap)


def sparse_static_gate(st: SparseStep, frame: torch.Tensor, status: torch.Tensor):
    """The overflow gate of the static forward on `frame` (a copy of the peer-visible frame), after the frame barrier
    that carried every rank's overflow word into ``status_array``. Queued before this rank's next barrier on the block:
    no peer can overwrite the status array before the gate has read it."""
    from .sharded import static_gate
    lib = _lib.load()
    rk = st.rk
    gb = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
    static_gate(st.s, rk.plan.world * st.cap, rk.cand[:gb], st.img, frame, status, flags=rk.status_array,
                error_word=rk.err_word)


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

    def __init__(self, plan: ShardPlan, device, W, H, exchange: Exchange, depth: int = 2, alpha: bool = False,
                 camera: bool = False, device_epoch: bool = False):
        self.all = []
        for k in range(depth):
            rk = SparseRank(plan, device, W, H, exchange=exchange, alpha=alpha, camera=camera)
            rk.index = k
            rk.device_epoch = bool(device_epoch)   # a static module: device-epoch barriers only, apply_weights included
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


def _preprocess_and_order(rk: SparseRank, pool: SparsePool, rs, means3D, sh, colors_precomp, opacities, scales, rotations,
                          cov3Ds_precomp, raw_rest=None, grad_mask=None):
    """preprocess + push -- barrier with the count row -- order, redone with the exact capacity while a segment
    overflows; then the capacity of the next step. Returns (step, num_rendered of this rank, largest segment)."""
    while True:
        st = sparse_preprocess(rk, rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                               pool.cap, raw_rest, grad_mask)
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
    pool.cap = next_capacity(max_count, rk.cap_alloc)
    return st, R, max_count


def apply_weights_walk(st: SparseStep, image_weights: torch.Tensor, acc: torch.Tensor, deterministic: bool = False):
    """Semantic tracing of the owned tiles of the candidate cloud into the zeroed rows `acc` [world*cap, 12]: weights in
    floats 0..CH-1, the count as int32 bits in float GSR_SPARSE_AW_CNT_SLOT (so that sparse_return carries it exactly).
    Deterministic mode reduces the weights into a packed zeroed [world*cap, CH] buffer and copies them into the rows."""
    from .sharded import owner_apply_weights
    rk = st.rk
    M = rk.plan.world * st.cap
    CH = int(image_weights.size(0))
    get = lambda name, n, dtype, grow: rk.get(name, n, dtype, grow)
    weights = rk.get("aw_det_weights", M * CH, torch.float32, grow=1.25).view(M, CH).zero_() if deterministic else acc
    owner_apply_weights(st.s, rk.plan.owner(), M, st.R, rk.cand, st.radii_cand, _f32c(image_weights, rk.device), weights,
                        CH if deterministic else ACC_STRIDE, acc.view(torch.int32)[:, AW_CNT_SLOT], ACC_STRIDE, get,
                        deterministic)
    if deterministic:
        acc[:, :CH].copy_(weights)


def apply_weights_gather(st: SparseStep, weights: torch.Tensor, cnt: torch.Tensor):
    """Owner side, after the return barrier: weights [n, CH] += and cnt [n] += the returned rows of each owned Gaussian,
    in ascending rank order."""
    lib = _lib.load()
    rk = st.rk
    CH = int(weights.size(1)) if weights.dim() > 1 else 1
    with torch.cuda.device(rk.device):
        stream = C.c_void_p(torch.cuda.current_stream(rk.device).cuda_stream)
        gb = lib.gsr_sparse_candidate_bytes(rk.plan.world, st.cap)
        _lib.check(lib.gsr_sparse_apply_weights_gather(C.byref(st.cplan), _ptr(rk.local), rk.local_bytes, _ptr(rk.cand), gb,
                                                       st.n, CH, _ptr(weights), _ptr(cnt), stream),
                   "gsr_sparse_apply_weights_gather")


def sparse_apply_weights(pool: SparsePool, rs, means3D, opacities, scales, rotations, cov3Ds_precomp, image_weights,
                         weights, cnt, deterministic: bool = False):
    """One view of semantic tracing with the sparse exchange (arguments checked by the caller): preprocess + push --
    barrier -- order (as the forward) -> walk of the owned tiles into zeroed candidate rows -> return -- barrier --
    gather into this rank's `weights` / `cnt`. A rank without owned tile rows or instances still takes part in every
    barrier. The workspace goes back to the pool before returning. The gather adds in ascending rank order, so
    `deterministic` only changes the walk."""
    rk = pool.take()
    empty = torch.empty(0, dtype=torch.float32, device=means3D.device)
    _mark("start")
    try:
        # this rank's means3D stands in the colors_precomp slot, as on one GPU: the colours are never used
        st, _, _ = _preprocess_and_order(rk, pool, rs, means3D, empty, means3D, opacities, scales, rotations,
                                         cov3Ds_precomp)
        M = rk.plan.world * st.cap
        acc = rk.get("acc", M * ACC_STRIDE, torch.float32, grow=1.25).view(M, ACC_STRIDE).zero_()
        apply_weights_walk(st, image_weights, acc, deterministic)
        _mark("walk")
        sparse_return(st, acc)
        peer_barrier(rk)
        _mark("return+barrier")
        apply_weights_gather(st, weights, cnt)
        _mark("gather")
    finally:
        pool.give(rk)


class _SparseShardedRasterize(torch.autograd.Function):
    """Sparse exchange; `depth_grad`, `raw_rest`, `return_alpha` and the camera inputs as in sharded._ShardedRasterize
    (the pool must have been built with the alpha plane / camera slots)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, pool, exchange,
                deterministic=False, depth_grad=False, raw_rest=None, return_alpha=False, viewmatrix=None,
                projmatrix=None, campos=None, grad_mask=None):
        rk0 = pool.all[0]
        if (return_alpha and rk0.planes != 5) or (viewmatrix is not None and not rk0.camera):
            raise RuntimeError("return_alpha / camera gradients need a SparsePool built with alpha=True / camera=True")
        rk = pool.take()
        device = means3D.device
        _mark("start")
        try:
            st, R, max_count = _preprocess_and_order(rk, pool, rs, means3D, sh, colors_precomp, opacities, scales,
                                                     rotations, cov3Ds_precomp, raw_rest, grad_mask)
        except BaseException:
            pool.give(rk)                                       # a failed forward must not leak its workspace
            raise
        weakref.finalize(st, pool.give, rk)
        # Every pixel has exactly one writer (the owner of its tile row; empty tiles are written too), so the frame needs
        # no zero-fill -- and must not get one: a faster peer may already have stored its rows here.
        frame = rk.frame
        sparse_render(st, frame[:3], frame[3:4])
        if return_alpha:   # every pixel of the alpha plane has one writer too: the owner of its tile row
            sparse_alpha(st, frame[4:5])
        _mark("bin+blend")
        frame_broadcast(rk)
        peer_barrier(rk)
        out = frame.clone()                                 # the peer-visible frame is overwritten by the next step
        _mark("frame broadcast+barrier")
        ctx.st, ctx.exchange, ctx.deterministic, ctx.depth_grad = st, exchange, deterministic, bool(depth_grad)
        ctx.return_alpha, ctx.camera_grad, ctx.rs = bool(return_alpha), viewmatrix is not None, rs
        if ctx.depth_grad or ctx.return_alpha:   # None = no gradient for that output (see sharded._ShardedRasterize)
            ctx.set_materialize_grads(False)
        radii = rk.radii_local[:rk.plan.count].clone()
        ctx.mark_non_differentiable(radii)
        _SparseShardedRasterize.last = dict(R=R, cap=st.cap, max_count=max_count)
        if return_alpha:
            return out[:3], radii, out[3:4], out[4:5]
        return out[:3], radii, out[3:4]

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_alpha=None):
        from .sharded import CAM_ROW, camera_grads_like, camera_row, combine_camera_rows
        st, exchange = ctx.st, ctx.exchange
        if st is None:
            raise RuntimeError("the sharded rasterizer's backward can run once (its workspace went back to the pool)")
        _mark("loss")
        grad_depth = grad_depth if ctx.depth_grad else None
        if grad_out_color is None:   # depth_grad / return_alpha: a loss on the depth or alpha alone
            grad_out_color = torch.zeros(3, st.rk.H, st.rk.W, dtype=torch.float32, device=st.rk.device)
        acc = sparse_backward_render(st, grad_out_color, ctx.deterministic, grad_depth, grad_alpha)
        _mark("blend backward")
        sparse_return(st, acc)
        peer_barrier(st.rk)
        _mark("return push+barrier")
        cam_grads = (None, None, None)
        if ctx.camera_grad:
            row, cam = camera_row(st.n, st.rk.device)
            grads = sparse_backward_preprocess(st, grad_depth is not None, cam)
            camera_put(st.rk, row)
            peer_barrier(st.rk)
            # read before this rank's next barrier on the block: no peer can store into the slots again until then
            cam_grads = camera_grads_like(combine_camera_rows(st.rk.cam_slots[:, :CAM_ROW]), ctx.rs)
            _mark("camera put+barrier")
        else:
            grads = sparse_backward_preprocess(st, grad_depth is not None)
        grads, d_rest = grads_in_slots(grads, len(st.inputs) == 8)
        _mark("gather+preprocess backward")
        ctx.st = None   # the workspace goes back to the pool now, not when the output tensors die
        return (*grads, None, None, None, None, None, d_rest, None, *cam_grads, None)


class _SparseShardedRasterizeStatic(torch.autograd.Function):
    """_SparseShardedRasterize for a fixed instance capacity and segment capacity (three more inputs: `capacity`,
    `seg_cap` and the device `status` int32[4]): no redo loop, no pinned words, no host wait, device-epoch barriers (the
    pool must be built with device_epoch=True). The frame barrier carries this rank's overflow word to every rank and the
    gate empties the output frame everywhere when any rank overflowed. The backward is _SparseShardedRasterize's with
    R = capacity, on scratch buffers of its own (sharded.StaticScratch)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, pool, exchange,
                deterministic=False, depth_grad=False, raw_rest=None, return_alpha=False, viewmatrix=None,
                projmatrix=None, campos=None, capacity=1, seg_cap=1, status=None, grad_mask=None):
        from .sharded import StaticScratch
        rk0 = pool.all[0]
        if (return_alpha and rk0.planes != 5) or (viewmatrix is not None and not rk0.camera) or not rk0.device_epoch:
            raise RuntimeError("the static sparse forward needs a SparsePool built with device_epoch=True (and alpha=True / "
                               "camera=True for return_alpha / camera gradients)")
        rk = pool.take()
        try:
            st = sparse_preprocess(rk, rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                   seg_cap, raw_rest, grad_mask)
            st.rk = StaticScratch(rk)                       # scratch of its own, never grown by apply_weights
            peer_barrier(rk, with_row=True)                # counts + barrier: every push has landed
            sparse_order_static(st, capacity)
        except BaseException:
            pool.give(rk)
            raise
        weakref.finalize(st, pool.give, rk)
        frame = rk.frame                                    # one writer per pixel: no zero-fill (see the default path)
        sparse_render_static(st, frame[:3], frame[3:4], status)
        if return_alpha:
            sparse_alpha(st, frame[4:5])
        frame_broadcast(rk)
        peer_barrier(rk, status_word=status[1:2])           # this rank's overflow word -> every rank's status array
        out = frame.clone()
        sparse_static_gate(st, out, status)
        ctx.st, ctx.exchange, ctx.deterministic, ctx.depth_grad = st, exchange, deterministic, bool(depth_grad)
        ctx.return_alpha, ctx.camera_grad, ctx.rs = bool(return_alpha), viewmatrix is not None, rs
        if ctx.depth_grad or ctx.return_alpha:
            ctx.set_materialize_grads(False)
        radii = rk.radii_local[:rk.plan.count].clone()
        ctx.mark_non_differentiable(radii)
        if return_alpha:
            return out[:3], radii, out[3:4], out[4:5]
        return out[:3], radii, out[3:4]

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_alpha=None):
        return (*_SparseShardedRasterize.backward(ctx, grad_out_color, grad_radii, grad_depth, grad_alpha), None, None,
                None)
