"""Gaussian-sharded multi-GPU rasterizer (BASELINE config 4, SURVEY.md 8(e)).

The reference has no multi-GPU rasterizer; this is the exact decomposition of the single-GPU pipeline over
``world`` ranks, one process per GPU:

  * rank g owns the Gaussians ``[g*L, g*L + n_g)`` (L = ceil(P/world)): parameters, optimizer state and the
    per-Gaussian stages (preprocess forward, fused preprocess backward) stay on the owner;
  * rank g owns the tile rows ``ty % world == g``: binning, blending and the blending backward run per tile owner;
  * three collectives join the two decompositions (all on the compute stream, issued by ``torch.distributed``):
      forward   ALL-GATHER   the 48-B splat records of every shard, in place (a record carries its radius and its
                             depth key, so nothing else has to travel)
                ALL-REDUCE   sum of the zero-initialised [4,H,W] frames (one writer per pixel: exact)
      backward  REDUCE-SCATTER  the [P,12] 2-D gradient accumulators back to the index owners

Because every P-sized array is indexed by GLOBAL Gaussian index, the gathered state equals the single-GPU state:
images, radii, n_contrib and the per-tile lists are bit-identical to ``GaussianRasterizer`` on one GPU (asserted in
tests/test_sharded.py); gradients agree to the usual float tolerance (the
order of the atomic sums differs).

The step functions (``shard_preprocess`` ... ``shard_backward_preprocess``) are thin wrappers of the C-ABI entry
points and can also be driven for several *virtual* ranks on one GPU, which is how the single-GPU test covers the
ownership logic.
"""
from __future__ import annotations

import ctypes as C
import weakref
import warnings
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib
from .rasterizer import (GaussianRasterizationSettings, _f32c, _geometry_bytes, _make_cloud, _make_settings,
                         _pinned_i32, _ptr, mark_visible)

ACC_STRIDE = 12  # floats per Gaussian in the 2-D gradient accumulators (csrc/common.cuh)


class ShardPlan(NamedTuple):
    """Index/tile ownership of one rank. ``P_total`` is the real cloud size, ``P_pad = slice_len * world`` the size
    of every gathered array (the tail of the last slice is marked culled)."""
    P_total: int
    world: int
    rank: int

    @property
    def slice_len(self) -> int:
        return (self.P_total + self.world - 1) // self.world if self.P_total > 0 else 0

    @property
    def P_pad(self) -> int:
        return self.slice_len * self.world

    @property
    def base(self) -> int:
        return self.rank * self.slice_len

    @property
    def count(self) -> int:
        """Number of real Gaussians this rank owns."""
        return max(0, min(self.P_total, self.base + self.slice_len) - self.base)

    def owned_tile_rows(self, H: int):
        gy = (H + 15) // 16
        return list(range(self.rank, gy, self.world))

    def owner(self) -> "_lib.TileOwner":
        return _lib.TileOwner(self.world, self.rank)


def shard_slice(t: torch.Tensor, plan: ShardPlan) -> torch.Tensor:
    """The rows of a full per-Gaussian tensor that `plan.rank` owns."""
    return t[plan.base:plan.base + plan.count]


# ---------------------------------------------------------------------------------------------------------
# collectives (backend-agnostic host logic; NCCL on GPUs, gloo in the CPU tests)
# ---------------------------------------------------------------------------------------------------------
def init_distributed(backend: str = "nccl", device: Optional[torch.device] = None):
    """``init_process_group`` from the torchrun environment with the one setting this path needs.

    ProcessGroupNCCL by default calls ``record_stream`` on every tensor a collective touches; the workspaces here are
    several hundred MB, freed and re-allocated every step, and the deferred frees cost a large share of a step at
    config 3. All collectives of this path are synchronous on the compute stream, so
    stream recording is not needed: TORCH_NCCL_AVOID_RECORD_STREAMS=1 (must be set before the group is created)."""
    import os
    import torch.distributed as dist
    os.environ.setdefault("TORCH_NCCL_AVOID_RECORD_STREAMS", "1")
    if dist.is_initialized():
        return
    if backend == "nccl":
        if device is None:
            device = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
        torch.cuda.set_device(device)
        dist.init_process_group("nccl", device_id=device)
    else:
        dist.init_process_group(backend)



class Exchange:
    """The three collectives of the sharded path over a ``torch.distributed`` process group."""

    def __init__(self, group=None):
        import torch.distributed as dist
        self.dist = dist
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.backend = dist.get_backend(group)

    def all_gather_inplace(self, total: torch.Tensor):
        """`total` is [world * n, ...]; rank r has filled rows [r*n, (r+1)*n). On return every rank has all rows."""
        n = total.shape[0] // self.world
        mine = total[self.rank * n:(self.rank + 1) * n]
        if self.backend == "nccl":
            self.dist.all_gather_into_tensor(total, mine, group=self.group)  # in place: send buffer = own slot
        else:  # gloo has no in-place flat all-gather
            parts = [torch.empty_like(mine) for _ in range(self.world)]
            self.dist.all_gather(parts, mine.clone(), group=self.group)
            for r, p in enumerate(parts):
                total[r * n:(r + 1) * n].copy_(p)

    def barrier(self, device):
        """Stream-ordered cross-rank barrier: a 4-byte all-reduce. Its completion on this rank implies every rank's
        earlier work on its compute stream (in particular its peer stores) has finished."""
        if getattr(self, "_flag", None) is None or self._flag.device != device:
            self._flag = torch.zeros(1, dtype=torch.int32, device=device)
        self.dist.all_reduce(self._flag, group=self.group)

    def all_reduce_sum(self, t: torch.Tensor):
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM, group=self.group)

    def all_to_all_single(self, out: torch.Tensor, inp: torch.Tensor, out_splits, in_splits):
        """Uneven all-to-all along dim 0: rank r receives `out_splits[q]` rows from every rank q, in rank order, and
        sends `in_splits[d]` rows of `inp` to rank d (the row moves of shard_rebalance.rebalance)."""
        if self.world == 1:
            out.copy_(inp)
            return
        self.dist.all_to_all_single(out, inp, output_split_sizes=list(out_splits), input_split_sizes=list(in_splits),
                                    group=self.group)

    def broadcast(self, t: torch.Tensor, src: int = 0):
        """`t` of group rank `src` on every rank."""
        if self.world == 1:
            return
        g = src if self.group is None else self.dist.get_global_rank(self.group, src)
        self.dist.broadcast(t, g, group=self.group)

    def reduce_scatter_sum(self, total: torch.Tensor, out: torch.Tensor):
        """out[n, ...] = sum over ranks of total[rank*n:(rank+1)*n]."""
        if self.backend == "nccl":
            self.dist.reduce_scatter_tensor(out, total, op=self.dist.ReduceOp.SUM, group=self.group)
        else:  # gloo: no reduce-scatter
            tmp = total.clone()
            self.dist.all_reduce(tmp, op=self.dist.ReduceOp.SUM, group=self.group)
            n = out.shape[0]
            out.copy_(tmp[self.rank * n:(self.rank + 1) * n])

    def reduce_scatter_ordered(self, total: torch.Tensor, out: torch.Tensor):
        """reduce_scatter_sum with a fixed summation order: every rank's slice comes here whole (all-to-all) and the
        slices are added in ascending rank order with plain tensor adds, so the result is the same bits on every call
        (NCCL's reduce-scatter does not promise an order). For the float sums of deterministic mode."""
        n = out.shape[0]
        if self.world == 1:
            out.copy_(total[:n])
            return
        recv = torch.empty((self.world,) + tuple(out.shape), dtype=out.dtype, device=out.device)
        send = total[:self.world * n].contiguous()
        if self.backend == "nccl":
            self.dist.all_to_all_single(recv, send, group=self.group)
        else:
            try:
                self.dist.all_to_all_single(recv, send, group=self.group)
            except (RuntimeError, NotImplementedError):   # a gloo build without all-to-all: gather and keep own slice
                parts = [torch.empty_like(send) for _ in range(self.world)]
                self.dist.all_gather(parts, send, group=self.group)
                for r, p in enumerate(parts):
                    recv[r].copy_(p[self.rank * n:(self.rank + 1) * n])
        out.copy_(recv[0])
        for r in range(1, self.world):
            out.add_(recv[r])


# ---------------------------------------------------------------------------------------------------------
# peer-mapped geometry workspaces (fused preprocess + all-gather over NVLink)
# ---------------------------------------------------------------------------------------------------------
class _RawCuda:
    """Zero-copy torch view of raw device memory (``__cuda_array_interface__``)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class PeerWorkspace:
    """One geometry workspace per rank, each mapped into every process of the group (CUDA IPC): `ptrs[r]` is rank
    r's buffer as seen from here. Created collectively (every rank must call with the same size, in the same order)."""

    def __init__(self, nbytes: int, exchange: Exchange, device: torch.device):
        lib = _lib.load()
        self.nbytes, self.world, self.rank = nbytes, exchange.world, exchange.rank
        own = C.c_void_p()
        handle = C.create_string_buffer(64)
        with torch.cuda.device(device):
            _lib.check(lib.gsr_peer_alloc(nbytes, C.byref(own), handle), "gsr_peer_alloc")
            handles = [None] * self.world
            exchange.dist.all_gather_object(handles, bytes(handle.raw), group=exchange.group)
            self.ptrs = []
            for r, h in enumerate(handles):
                if r == self.rank:
                    self.ptrs.append(own.value)
                else:
                    p = C.c_void_p()
                    _lib.check(lib.gsr_peer_open(C.create_string_buffer(h, 64), C.byref(p)), "gsr_peer_open")
                    self.ptrs.append(p.value)
        self.ptr_array = (C.c_void_p * self.world)(*self.ptrs)
        self.tensor = torch.as_tensor(_RawCuda(own.value, nbytes), device=device)  # the local buffer as uint8 tensor
        self.device = device

    def close(self):
        lib = _lib.load()
        with torch.cuda.device(self.device):
            torch.cuda.synchronize()
            for r, p in enumerate(self.ptrs):
                if p is not None and r != self.rank:
                    lib.gsr_peer_close(C.c_void_p(p))
            self.tensor = None
            lib.gsr_peer_free(C.c_void_p(self.ptrs[self.rank]))
        self.ptrs = [None] * self.world


class StepWorkspace:
    """Persistent device buffers of one in-flight forward/backward: the geometry workspace (peer-mapped when `peer` is
    given), radii, binning (grow-only), image state and the gradient accumulators. Re-using them across steps keeps
    the caching allocator out of the step: the sizes change with every camera (num_rendered), and several-hundred-MB
    blocks that come and go cost cudaMalloc/cudaFree stalls of milliseconds (measured: 3.0 vs 1.9 ms/step on 4 GPUs)."""

    def __init__(self, device, peer: Optional[PeerWorkspace] = None):
        self.device, self.peer = device, peer
        self.bufs: dict = {}
        self.index = 0

    def get(self, name: str, numel: int, dtype, grow: float = 1.0) -> torch.Tensor:
        t = self.bufs.get(name)
        if t is None or t.numel() < numel or t.dtype != dtype:
            t = self.bufs[name] = torch.empty(int(numel * grow) + 256, dtype=dtype, device=self.device)
        return t[:numel]

    def close(self):
        self.bufs.clear()
        if self.peer is not None:
            self.peer.close()
            self.peer = None


class WorkspacePool:
    """Free list of StepWorkspaces. A workspace is taken per forward and given back when that forward's buffers die
    (after its backward, or when its outputs are dropped), so several forwards may be alive at once (GaussianEditor
    renders twice per step before one backward). Every rank runs the same sequence, which keeps the pools aligned:
    peer workspace k on rank A is always paired with workspace k on rank B.

    Re-use of a peer workspace is safe without extra synchronisation: a rank starts the next preprocess only after
    its own step finished, and the last collective of a step (frame all-reduce / accumulator reduce-scatter) cannot
    complete here before every peer has finished the kernels that read its workspace."""

    def __init__(self, exchange: Exchange, geometry_bytes: int, p2p: bool):
        self.exchange, self.nbytes, self.p2p = exchange, geometry_bytes, p2p
        self.free: list = []
        self.all: list = []

    def take(self, device) -> StepWorkspace:
        if self.free:
            return self.free.pop(0)
        ws = StepWorkspace(device, PeerWorkspace(self.nbytes, self.exchange, device) if self.p2p else None)
        ws.index = len(self.all)
        self.all.append(ws)
        return ws

    def give(self, ws: StepWorkspace):
        self.free.append(ws)
        self.free.sort(key=lambda w: w.index)

    def close(self):
        for ws in self.all:
            ws.close()
        self.all, self.free = [], []


# ---------------------------------------------------------------------------------------------------------
# step functions = the C-ABI entry points
# ---------------------------------------------------------------------------------------------------------
class ShardBuffers:
    """Per-rank device state of one sharded forward (all arrays indexed by global Gaussian index)."""
    __slots__ = ("plan", "geom", "radii", "binning", "img", "R", "M", "W", "H", "inputs", "s", "own", "keep", "peer",
                 "ws", "grad_mask", "__weakref__")

    def alloc(self, name: str, numel: int, dtype, device, grow: float = 1.0) -> torch.Tensor:
        """A scratch buffer: from the persistent StepWorkspace when there is one, else from the caching allocator."""
        if self.ws is not None:
            return self.ws.get(name, numel, dtype, grow)
        return torch.empty(numel, dtype=dtype, device=device)


_mask_stand_in = {}


def mask_ptr(mask: torch.Tensor):
    """The pointer of a rank's grad_mask rows for the masked entry points, which reject NULL: an empty shard (whose
    mask has no storage) passes a 1-byte stand-in that nothing reads."""
    if mask.numel() > 0:
        return _ptr(mask)
    t = _mask_stand_in.get(mask.device)
    if t is None:
        t = _mask_stand_in[mask.device] = torch.zeros(1, dtype=torch.uint8, device=mask.device)
    return _ptr(t)


def _view_bytes(base: torch.Tensor, ptr: int, nbytes: int) -> torch.Tensor:
    off = ptr - base.data_ptr()
    return base[off:off + nbytes]


_rec_offset: dict = {}


def exchange_view(buf: ShardBuffers) -> torch.Tensor:
    """The splat records [P_pad, 48] (uint8 view onto the geometry workspace): the one array that is exchanged."""
    P = buf.plan.P_pad
    off = _rec_offset.get(P)
    if off is None:
        v = _lib.ExchangeView()
        _lib.check(_lib.load().gsr_view_exchange(_ptr(buf.geom), P, C.byref(v)), "gsr_view_exchange")
        off = _rec_offset[P] = v.records - buf.geom.data_ptr()
    return buf.geom[off:off + P * 48].view(P, 48)


def shard_preprocess(plan: ShardPlan, rs: GaussianRasterizationSettings, means3D, sh, colors_precomp, opacities,
                     scales, rotations, cov3Ds_precomp, *, geom: Optional[torch.Tensor] = None,
                     radii: Optional[torch.Tensor] = None, peer: Optional[PeerWorkspace] = None,
                     ws: Optional[StepWorkspace] = None, raw_rest: Optional[torch.Tensor] = None,
                     grad_mask: Optional[torch.Tensor] = None) -> ShardBuffers:
    """Stage 1: project this rank's Gaussians into its slice of the global arrays. `geom` / `radii` may be passed
    in to share one set of global arrays between virtual ranks of a single process. With `peer` (a PeerWorkspace of
    gsr_geometry_bytes(P_pad) bytes) the kernel pushes its records into every rank's workspace itself: no all-gather
    follows, only a barrier. `ws` (a StepWorkspace) supplies all scratch buffers persistently, its `peer` included.
    With `raw_rest` (features_rest [n,K,3]) the shard is the scene model's raw parameters (fused activations): `sh` is
    features_dc [n,1,3], `opacities` / `scales` / `rotations` are the logits, log-scales and raw rotations. With
    `grad_mask` (uint8 [n], this rank's rows) the masked twin writes each edited Gaussian's edit word into its record,
    for the masked blend backward of every tile owner."""
    lib = _lib.load()
    if ws is not None and ws.peer is not None:
        peer = ws.peer
    if not means3D.is_cuda:
        raise RuntimeError("the rasterizer needs CUDA tensors (there is no CPU path)")
    if means3D.size(0) != plan.count:
        raise RuntimeError(f"rank {plan.rank} owns {plan.count} Gaussians, got {means3D.size(0)}")
    device = means3D.device
    H, W = int(rs.image_height), int(rs.image_width)
    M = sh.size(1) if sh.numel() != 0 else 0
    if raw_rest is not None:
        M = 1 + raw_rest.size(1)
    buf = ShardBuffers()
    buf.plan, buf.M, buf.W, buf.H, buf.ws, buf.grad_mask = plan, M, W, H, ws, grad_mask
    with torch.cuda.device(device):
        means3D = _f32c(means3D, device); opacities = _f32c(opacities, device)
        sh = _f32c(sh, device); colors_precomp = _f32c(colors_precomp, device)
        scales = _f32c(scales, device); rotations = _f32c(rotations, device)
        cov3Ds_precomp = _f32c(cov3Ds_precomp, device)
        buf.inputs = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
        if raw_rest is not None:   # a slice whose rows start off a 16-byte boundary is cloned by _f32c
            buf.inputs = buf.inputs + (_f32c(raw_rest, device),)
        gbytes = _geometry_bytes(lib, plan.P_pad)
        buf.peer = peer
        if peer is not None:
            if peer.nbytes < gbytes:
                raise RuntimeError(f"peer workspace too small: {peer.nbytes} < {gbytes}")
            geom = peer.tensor
        buf.geom = geom if geom is not None else buf.alloc("geom", gbytes, torch.uint8, device)
        buf.radii = radii if radii is not None else buf.alloc("radii", plan.P_pad, torch.int32, device)
        buf.keep = []
        s = buf.s = _make_settings(rs, M, device, buf.keep)   # one settings struct for all five stage calls
        buf.own = plan.owner()
        c = _shard_cloud(plan.count, buf.inputs)
        raw = "_raw" if len(buf.inputs) == 8 else ""
        masked = () if grad_mask is None else (mask_ptr(grad_mask),)
        sfx = raw + ("_masked" if masked else "")
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        if peer is not None:
            _lib.check(getattr(lib, "gsr_shard_preprocess_p2p" + sfx)(
                C.byref(s), C.byref(c), plan.P_pad, plan.base, plan.slice_len, peer.ptr_array, plan.world, plan.rank,
                peer.nbytes, _ptr(buf.radii), *masked, st), "gsr_shard_preprocess_p2p" + sfx)
        else:
            _lib.check(getattr(lib, "gsr_shard_preprocess" + sfx)(
                C.byref(s), C.byref(c), plan.P_pad, plan.base, plan.slice_len, _ptr(buf.geom), gbytes,
                _ptr(buf.radii), *masked, st), "gsr_shard_preprocess" + sfx)
    return buf


def _shard_cloud(n: int, inputs):
    """The C struct of a shard's inputs: gsr_cloud, or gsr_raw_cloud when `inputs` carries features_rest (8 entries)."""
    (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp) = inputs[:7]
    if len(inputs) == 8:
        return _lib.RawCloud(n, _ptr(means3D), _ptr(opacities), _ptr(sh), _ptr(inputs[7]), _ptr(scales), _ptr(rotations))
    return _make_cloud(n, means3D, opacities, sh, colors_precomp, scales, rotations, cov3Ds_precomp)


def preprocess_grads(lib, n: int, M: int, inputs, device, call):
    """Gradient buffers of a shard's fused preprocess backward; `call(cloud, grads, raw)` runs the entry point (not for
    n == 0). Activated inputs: the 8 tensors of the reference's slot order (means3D, means2D, sh, colors, opacity,
    scales, rotations, cov3D). Raw inputs (features_rest present): means3D, means2D, opacity_logits, features_dc,
    features_rest, log_scales, raw_rotations."""
    f32 = dict(dtype=torch.float32, device=device)
    raw = len(inputs) == 8
    with torch.cuda.device(device):
        if raw:
            d_m3 = torch.empty(n, 3, **f32); d_m2 = torch.empty(n, 3, **f32); d_op = torch.empty(n, 1, **f32)
            d_dc = torch.empty(n, 1, 3, **f32); d_rest = torch.empty(n, M - 1, 3, **f32)
            d_sc = torch.empty(n, 3, **f32); d_ro = torch.empty(n, 4, **f32)
            if n > 0:
                call(_shard_cloud(n, inputs), _lib.RawGrads(_ptr(d_m3), _ptr(d_m2), _ptr(d_op), _ptr(d_dc),
                                                            _ptr(d_rest), _ptr(d_sc), _ptr(d_ro)), True)
            return (d_m3, d_m2, d_op, d_dc, d_rest, d_sc, d_ro)
        dL_dmeans3D = torch.empty(n, 3, **f32); dL_dmeans2D = torch.empty(n, 3, **f32)
        dL_dcolors = torch.empty(n, 3, **f32); dL_dopacity = torch.empty(n, 1, **f32)
        dL_dcov3D = torch.empty(n, 6, **f32); dL_dsh = torch.empty(n, M, 3, **f32)
        dL_dscales = torch.empty(n, 3, **f32); dL_drotations = torch.empty(n, 4, **f32)
        if n > 0:
            call(_shard_cloud(n, inputs), _lib.Grads(_ptr(dL_dmeans3D), _ptr(dL_dmeans2D), _ptr(dL_dcolors),
                                                     _ptr(dL_dopacity), _ptr(dL_dcov3D), _ptr(dL_dsh),
                                                     _ptr(dL_dscales), _ptr(dL_drotations)), False)
            if inputs[4].numel() == 0:
                dL_dscales.zero_(); dL_drotations.zero_()
    return (dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D)


def shard_order(buf: ShardBuffers) -> int:
    """Stage 2 (after the all-gather): radii of all Gaussians, owned-tile counts, depth order, scan. Returns this
    rank's instance count (one stream synchronisation to read it)."""
    lib = _lib.load()
    device = buf.geom.device
    with torch.cuda.device(device):
        s, own = buf.s, buf.own
        stream = torch.cuda.current_stream(device)
        pinned = _pinned_i32(device)
        _lib.check(lib.gsr_shard_order(C.byref(s), C.byref(own), buf.plan.P_pad, _ptr(buf.geom), buf.geom.numel(),
                                       _ptr(buf.radii), C.c_void_p(pinned.data_ptr()),
                                       C.c_void_p(stream.cuda_stream)), "gsr_shard_order")
        stream.synchronize()
        buf.R = int(pinned[0])
    return buf.R


def shard_render(buf: ShardBuffers, color: torch.Tensor, depth: torch.Tensor):
    """Stage 3: bin + blend the owned tiles into `color` [3,H,W] / `depth` [1,H,W] (zero elsewhere: caller zero-fills)."""
    lib = _lib.load()
    device = buf.geom.device
    with torch.cuda.device(device):
        s, own = buf.s, buf.own
        P, R, W, H = buf.plan.P_pad, buf.R, buf.W, buf.H
        bbytes = lib.gsr_binning_bytes(P, R, W, H) if R > 0 else 0
        buf.binning = buf.alloc("binning", bbytes, torch.uint8, device, grow=1.25)
        ibytes = lib.gsr_image_bytes(W, H)
        buf.img = buf.alloc("img", ibytes, torch.uint8, device)
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(lib.gsr_shard_render(C.byref(s), C.byref(own), P, R, _ptr(buf.geom), buf.geom.numel(),
                                        _ptr(buf.binning), bbytes, _ptr(buf.img), ibytes, _ptr(buf.radii),
                                        _ptr(color), _ptr(depth), st), "gsr_shard_render")


def shard_alpha(buf: ShardBuffers, alpha: torch.Tensor):
    """After shard_render: alpha = 1 - final_T on the owned tile rows of `alpha` [1,H,W] (other rows untouched)."""
    lib = _lib.load()
    device = buf.geom.device
    with torch.cuda.device(device):
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(lib.gsr_shard_alpha_image(C.byref(buf.own), _ptr(buf.img), buf.img.numel(), buf.W, buf.H, _ptr(alpha),
                                             st), "gsr_shard_alpha_image")


# ---- fixed-capacity (static) forward: no host copy, no host wait ---------------------------------------------------
STATUS_WORDS = 4   # status = {R of this rank, overflow (any rank), largest segment (sparse), barrier error (sparse)}


class StaticScratch:
    """A StepWorkspace or SparseRank seen through its ``get`` with every scratch name prefixed ``static_``: the
    fixed-capacity step keeps buffers of its own, so that an ``apply_weights`` (host-sized, grow-only scratch) can never
    re-allocate a buffer a captured CUDA graph still points to. Every other attribute is the wrapped object's."""

    def __init__(self, inner):
        self.inner = inner

    def get(self, name: str, numel: int, dtype, grow: float = 1.0) -> torch.Tensor:
        return self.inner.get("static_" + name, numel, dtype, grow)

    def __getattr__(self, name):
        return getattr(self.inner, name)


def shard_order_static(buf: ShardBuffers, capacity: int):
    """shard_order without the readback (gsr_shard_order_static): R stays on the device, and ``buf.R = capacity`` sizes
    the binning and every backward behind it."""
    lib = _lib.load()
    device = buf.geom.device
    with torch.cuda.device(device):
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(lib.gsr_shard_order_static(C.byref(buf.s), C.byref(buf.own), buf.plan.P_pad, _ptr(buf.geom),
                                              buf.geom.numel(), _ptr(buf.radii), st), "gsr_shard_order_static")
    buf.R = int(capacity)


def render_static(s, own, P: int, capacity: int, geom: torch.Tensor, radii: torch.Tensor, color: torch.Tensor,
                  depth: torch.Tensor, status: torch.Tensor, get, counts: Optional[torch.Tensor] = None, world: int = 0,
                  seg_cap: int = 0):
    """gsr_shard_render_static of a P-record workspace `geom` for `capacity` instances; returns (binning, img) from
    `get(name, numel, dtype, grow)`. `counts` (the sparse count matrix, with `world` and `seg_cap`) adds the segment
    check to ``status``."""
    lib = _lib.load()
    device = geom.device
    W, H = int(s.image_width), int(s.image_height)
    with torch.cuda.device(device):
        bbytes = lib.gsr_binning_bytes(P, capacity, W, H)
        binning = get("binning", bbytes, torch.uint8, 1.0)
        ibytes = lib.gsr_image_bytes(W, H)
        img = get("img", ibytes, torch.uint8, 1.0)
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(lib.gsr_shard_render_static(C.byref(s), C.byref(own), P, capacity, _ptr(geom), geom.numel(),
                                               _ptr(binning), bbytes, _ptr(img), ibytes, _ptr(radii), _ptr(color),
                                               _ptr(depth), _ptr(status), _ptr(counts), world, seg_cap, st),
                   "gsr_shard_render_static")
    return binning, img


def shard_render_static(buf: ShardBuffers, color: torch.Tensor, depth: torch.Tensor, status: torch.Tensor):
    """shard_render for the capacity of shard_order_static: ``status`` (device int32[4]) gets {R, R > capacity, 0, 0}
    and an overflowing rank's owned tiles are rendered empty."""
    device = buf.geom.device
    buf.binning, buf.img = render_static(buf.s, buf.own, buf.plan.P_pad, buf.R, buf.geom, buf.radii, color, depth,
                                         status, lambda name, n, dtype, grow: buf.alloc(name, n, dtype, device, grow))


def static_gate(s, P: int, geom: torch.Tensor, img: torch.Tensor, frame: torch.Tensor, status: torch.Tensor,
                flags: Optional[torch.Tensor] = None, flag_sum: Optional[torch.Tensor] = None,
                error_word: Optional[torch.Tensor] = None):
    """gsr_shard_static_gate: if any rank overflowed (`flags` int32 [world] or the all-reduced float `flag_sum` [1]),
    `frame` [planes,H,W] becomes the empty frame and this rank's tiles are emptied, so every backward returns zeros.
    status[1] = the global flag, status[3] = the barrier error word."""
    lib = _lib.load()
    device = geom.device
    with torch.cuda.device(device):
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(lib.gsr_shard_static_gate(C.byref(s), P, _ptr(geom), geom.numel(), _ptr(img), img.numel(),
                                             _ptr(flags), 0 if flags is None else int(flags.numel()), _ptr(flag_sum),
                                             _ptr(error_word), _ptr(frame), int(frame.size(0)), _ptr(status), st),
                   "gsr_shard_static_gate")


def static_status_error(status, capacity: int, segment_capacity: Optional[int], rank: int) -> Optional[str]:
    """The message ``check_capacity`` raises for the host copy `status` [4] of a static sharded forward, or None."""
    R, over, max_count, err = (int(v) for v in status)
    if err:
        return (f"rank {rank}: a peer barrier of the sparse exchange timed out (a peer rank died, hung or runs a "
                "different step sequence); the exchanged data of this step are not valid")
    if not over:
        return None
    if R > capacity:
        why = f"this rank's instance count R={R} exceeds static_capacity={capacity}"
    elif segment_capacity is not None and max_count > segment_capacity:
        why = f"a sparse segment of {max_count} records exceeds segment_capacity={segment_capacity}"
    else:
        why = f"another rank's instance count exceeds static_capacity={capacity} (this rank's R={R})"
    return f"rank {rank}: {why}: the frame was rendered empty on every rank; re-size and rebuild the module"


def owner_backward_render(s, own, P: int, R: int, geom: torch.Tensor, binning: torch.Tensor, img: torch.Tensor,
                          grad_out_color: torch.Tensor, acc: torch.Tensor, deterministic: bool, get,
                          grad_depth: Optional[torch.Tensor] = None, grad_alpha: Optional[torch.Tensor] = None,
                          masked: bool = False):
    """gsr_shard_backward_render (or its deterministic form) of the owned tiles of a P-record workspace into
    acc [P, 12]; `get(name, numel, dtype, grow)` supplies the deterministic scratch. With `grad_depth` [1,H,W]
    (gsr_shard_backward_render_depth) float 9 of each row also gets dL/dz. With `grad_alpha` [1,H,W]
    (gsr_shard_backward_render_alpha, `grad_depth` optional) the alpha image's gradient enters too. `masked`: the
    records come from a masked preprocess, and gsr_shard_backward_render_masked skips the unedited splats' work (their
    rows stay +0.0)."""
    lib = _lib.load()
    device = geom.device
    with torch.cuda.device(device):
        grad_out_color = _f32c(grad_out_color, device)
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        if masked:
            grad_alpha = None if grad_alpha is None else _f32c(grad_alpha, device)
            grad_depth = None if grad_depth is None else _f32c(grad_depth, device)
            det, dbytes = None, 0
            if deterministic:
                dbytes = lib.gsr_deterministic_scratch_bytes(P, R, 0)
                det = get("det", dbytes, torch.uint8, 1.25)
            mbytes = lib.gsr_grad_mask_scratch_bytes(int(s.image_width), int(s.image_height))
            first = get("grad_mask_first", mbytes, torch.uint8, 1.0)
            _lib.check(lib.gsr_shard_backward_render_masked(
                C.byref(s), C.byref(own), P, R, _ptr(geom), geom.numel(), _ptr(binning), binning.numel(), _ptr(img),
                img.numel(), _ptr(grad_out_color), _ptr(grad_alpha), _ptr(grad_depth), _ptr(acc), acc.numel() * 4,
                _ptr(det), dbytes, _ptr(first), mbytes, st), "gsr_shard_backward_render_masked")
            return
        if grad_alpha is not None:
            grad_alpha = _f32c(grad_alpha, device)
            grad_depth = None if grad_depth is None else _f32c(grad_depth, device)
            det, dbytes = None, 0
            if deterministic:
                dbytes = lib.gsr_deterministic_scratch_bytes(P, R, 0)
                det = get("det", dbytes, torch.uint8, 1.25)
            _lib.check(lib.gsr_shard_backward_render_alpha(
                C.byref(s), C.byref(own), P, R, _ptr(geom), geom.numel(), _ptr(binning), binning.numel(), _ptr(img),
                img.numel(), _ptr(grad_out_color), _ptr(grad_alpha), _ptr(grad_depth), _ptr(acc), acc.numel() * 4,
                _ptr(det), dbytes, st), "gsr_shard_backward_render_alpha")
            return
        if grad_depth is not None:
            grad_depth = _f32c(grad_depth, device)
            args = (C.byref(s), C.byref(own), P, R, _ptr(geom), geom.numel(), _ptr(binning), binning.numel(),
                    _ptr(img), img.numel(), _ptr(grad_out_color), _ptr(grad_depth), _ptr(acc), acc.numel() * 4)
            det, dbytes = None, 0
            if deterministic:
                dbytes = lib.gsr_deterministic_scratch_bytes(P, R, 0)
                det = get("det", dbytes, torch.uint8, 1.25)
            _lib.check(lib.gsr_shard_backward_render_depth(*args, _ptr(det), dbytes, st),
                       "gsr_shard_backward_render_depth")
            return
        args = (C.byref(s), C.byref(own), P, R, _ptr(geom), geom.numel(), _ptr(binning), binning.numel(), _ptr(img),
                img.numel(), _ptr(grad_out_color), _ptr(acc), acc.numel() * 4)
        if deterministic:
            dbytes = lib.gsr_deterministic_scratch_bytes(P, R, 0)
            det = get("det", dbytes, torch.uint8, 1.25)
            _lib.check(lib.gsr_shard_backward_render_deterministic(*args, _ptr(det), dbytes, st),
                       "gsr_shard_backward_render_deterministic")
        else:
            _lib.check(lib.gsr_shard_backward_render(*args, st), "gsr_shard_backward_render")


def shard_backward_render(buf: ShardBuffers, grad_out_color: torch.Tensor, deterministic: bool = False,
                          grad_depth: Optional[torch.Tensor] = None,
                          grad_alpha: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Backward stage 1: this rank's tiles -> partial accumulators [P_pad, 12] (zero for untouched Gaussians). With
    `deterministic` each row is the same bits on every call (no float atomics). With `grad_depth` [1,H,W] the depth
    image's gradient enters too (dL/dz in float 9), with `grad_alpha` [1,H,W] the alpha image's. After a masked
    shard_preprocess only the edited Gaussians' rows are nonzero."""
    device = buf.geom.device
    acc = buf.alloc("acc", buf.plan.P_pad * ACC_STRIDE, torch.float32, device).view(buf.plan.P_pad, ACC_STRIDE)
    owner_backward_render(buf.s, buf.own, buf.plan.P_pad, buf.R, buf.geom, buf.binning, buf.img, grad_out_color, acc,
                          deterministic, lambda name, n, dtype, grow: buf.alloc(name, n, dtype, device, grow),
                          grad_depth, grad_alpha, buf.grad_mask is not None)
    return acc


CAM_ROW = 35   # one rank's camera-gradient partial: dL/dviewmatrix [16], dL/dprojmatrix [16], dL/dcampos [3]


def camera_row(n: int, device):
    """(row, gsr_camera_grads) of a shard of n Gaussians: the entry points write the partial into the zeroed `row`
    [CAM_ROW] (an empty shard is not called and keeps its zero row). The struct keeps its scratch alive in `_keep`."""
    lib = _lib.load()
    row = torch.zeros(CAM_ROW, dtype=torch.float32, device=device)
    cbytes = lib.gsr_camera_scratch_bytes(n)
    scratch = torch.empty(cbytes, dtype=torch.uint8, device=device)
    cam = _lib.CameraGrads(_ptr(row[:16]), _ptr(row[16:32]), _ptr(row[32:]), _ptr(scratch), cbytes)
    cam._keep = scratch
    return row, cam


def combine_camera_rows(rows: torch.Tensor) -> torch.Tensor:
    """The camera gradients of the whole cloud from the ranks' partials `rows` [world, CAM_ROW]: plain fp32 adds in
    ascending rank order, so every rank that holds the same rows gets the same bits (an all-reduce fixes no order). At
    world 1 the result is row 0 itself."""
    out = rows[0].clone()
    for r in range(1, rows.size(0)):
        out.add_(rows[r])
    return out


def camera_grads_like(total: torch.Tensor, rs) -> tuple:
    """A combined row as (dL/dviewmatrix, dL/dprojmatrix, dL/dcampos) shaped like the settings' camera arrays."""
    return (total[:16].reshape(rs.viewmatrix.shape), total[16:32].reshape(rs.projmatrix.shape),
            total[32:CAM_ROW].reshape(rs.campos.shape))


def shard_backward_preprocess(buf: ShardBuffers, acc_slice: torch.Tensor, depth: bool = False,
                              camera: Optional[_lib.CameraGrads] = None):
    """Backward stage 2 (after the reduce-scatter): gradients of this rank's Gaussians, reference slot order (or the
    raw parameters' order of GaussianRasterizer.forward_raw for a raw shard). `depth`: the rows carry dL/dz (the
    blending backward had a depth gradient). `camera` (from camera_row, activated shards only): this rank's camera
    partial is written too (gsr_shard_backward_preprocess_camera). After a masked shard_preprocess the masked twin
    writes +0.0 into every gradient of an unedited Gaussian (``buf.grad_mask`` as it holds now)."""
    lib = _lib.load()
    device = buf.geom.device
    plan = buf.plan

    def call(c, gr, raw):
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        args = (C.byref(buf.s), C.byref(c), plan.P_pad, plan.base, _ptr(buf.geom), buf.geom.numel(), _ptr(buf.radii),
                _ptr(acc_slice), C.byref(gr))
        if buf.grad_mask is not None:
            if raw:
                _lib.check(lib.gsr_shard_backward_preprocess_raw_masked(*args, int(depth), mask_ptr(buf.grad_mask), st),
                           "gsr_shard_backward_preprocess_raw_masked")
            else:
                _lib.check(lib.gsr_shard_backward_preprocess_masked(*args, int(depth), None, mask_ptr(buf.grad_mask),
                                                                    st), "gsr_shard_backward_preprocess_masked")
        elif camera is not None:
            _lib.check(lib.gsr_shard_backward_preprocess_camera(*args, int(depth), C.byref(camera), st),
                       "gsr_shard_backward_preprocess_camera")
        elif raw:
            _lib.check(lib.gsr_shard_backward_preprocess_raw(*args, int(depth), st), "gsr_shard_backward_preprocess_raw")
        elif depth:
            _lib.check(lib.gsr_shard_backward_preprocess_depth(*args, st), "gsr_shard_backward_preprocess_depth")
        else:
            _lib.check(lib.gsr_shard_backward_preprocess(*args, st), "gsr_shard_backward_preprocess")
    return preprocess_grads(lib, plan.count, buf.M, buf.inputs, device, call)


def owner_apply_weights(s, own, P: int, R: int, geom: torch.Tensor, radii: torch.Tensor, image_weights: torch.Tensor,
                        weights: torch.Tensor, w_stride: int, cnt: torch.Tensor, c_stride: int, get,
                        deterministic: bool = False):
    """gsr_shard_apply_weights: bin + walk the owned tiles of a P-record workspace `geom` (after the order stage),
    adding the hits of record i to weights[i*w_stride + ch] and cnt[i*c_stride]. `get(name, numel, dtype, grow)`
    supplies the binning and image scratch, sized from the settings `s` (not from a frame size fixed elsewhere).
    `deterministic` (gsr_shard_apply_weights_deterministic) needs packed weights, w_stride == CH."""
    lib = _lib.load()
    device = geom.device
    W, H = int(s.image_width), int(s.image_height)
    CH = int(image_weights.size(0))
    with torch.cuda.device(device):
        bbytes = lib.gsr_binning_bytes(P, R, W, H) if R > 0 else 0
        binning = get("binning", bbytes, torch.uint8, 1.25)
        ibytes = lib.gsr_image_bytes(W, H)
        img = get("img", ibytes, torch.uint8, 1.0)
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        args = (C.byref(s), C.byref(own), P, R, _ptr(geom), geom.numel(), _ptr(binning), bbytes, _ptr(img), ibytes,
                _ptr(radii), _ptr(image_weights), CH, _ptr(weights), w_stride, _ptr(cnt), c_stride)
        if deterministic:
            dbytes = lib.gsr_deterministic_scratch_bytes(P, R, CH)
            det = get("det", dbytes, torch.uint8, 1.25)
            _lib.check(lib.gsr_shard_apply_weights_deterministic(*args, _ptr(det), dbytes, st),
                       "gsr_shard_apply_weights_deterministic")
        else:
            _lib.check(lib.gsr_shard_apply_weights(*args, st), "gsr_shard_apply_weights")


def shard_apply_weights(buf: ShardBuffers, image_weights: torch.Tensor, weights_total: torch.Tensor,
                        cnt_total: torch.Tensor, deterministic: bool = False):
    """Semantic tracing of the owned tiles (after shard_order): adds into `weights_total` [P_pad, CH] float32 and
    `cnt_total` [P_pad] int32, indexed by global Gaussian index (the caller zero-fills them)."""
    device = buf.geom.device
    owner_apply_weights(buf.s, buf.own, buf.plan.P_pad, buf.R, buf.geom, buf.radii, _f32c(image_weights, device),
                        weights_total, int(image_weights.size(0)), cnt_total, 1,
                        lambda name, n, dtype, grow: buf.alloc(name, n, dtype, device, grow), deterministic)


def check_apply_weights_args(plan: ShardPlan, rs, means3D, weights, cnt, image_weights, scales, rotations,
                             cov3Ds_precomp) -> int:
    """The argument checks of ShardedGaussianRasterizer.apply_weights (this rank's rows), all made before any collective
    so that a bad argument raises here instead of leaving the peers waiting. Returns CH."""
    assert weights is not None
    assert cnt is not None
    assert image_weights is not None
    if ((scales is None or rotations is None) and cov3Ds_precomp is None) or (
            (scales is not None or rotations is not None) and cov3Ds_precomp is not None):
        raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
    if not means3D.is_cuda:
        raise RuntimeError("the rasterizer needs CUDA tensors (there is no CPU path)")
    if means3D.size(0) != plan.count:
        raise RuntimeError(f"rank {plan.rank} owns {plan.count} Gaussians, got {means3D.size(0)}")
    if not (weights.is_cuda and weights.dtype == torch.float32 and weights.is_contiguous()):
        raise RuntimeError("weights must be a contiguous float32 CUDA tensor (it is updated in place)")
    if not (cnt.is_cuda and cnt.dtype == torch.int32 and cnt.is_contiguous()):
        raise RuntimeError("cnt must be a contiguous int32 CUDA tensor (it is updated in place)")
    H, W = int(rs.image_height), int(rs.image_width)
    if image_weights.dim() != 3 or not 1 <= image_weights.size(0) <= 3 or tuple(image_weights.shape[1:]) != (H, W):
        raise RuntimeError(f"image_weights must be [CH, {H}, {W}] with CH in 1..3, got {tuple(image_weights.shape)}")
    CH = int(image_weights.size(0))
    if weights.numel() != plan.count * CH or (weights.dim() > 0 and weights.size(0) != plan.count):
        raise RuntimeError(f"weights must be this rank's [{plan.count}, {CH}] rows, got {tuple(weights.shape)}")
    if cnt.numel() != plan.count:
        raise RuntimeError(f"cnt must be this rank's [{plan.count}, 1] rows, got {tuple(cnt.shape)}")
    return CH


def dense_apply_weights(plan: ShardPlan, exchange: "Exchange", pool: "WorkspacePool", rs, means3D, opacities, scales,
                        rotations, cov3Ds_precomp, image_weights, weights, cnt, deterministic: bool = False):
    """One view of semantic tracing in the dense exchange: preprocess -> all-gather (or barrier) -> order -> walk of
    the owned tiles into zeroed [P_pad, CH] / [P_pad] buffers -> reduce-scatter of both (cnt stays int32) -> this
    rank's slices added into `weights` / `cnt`. `deterministic`: deterministic walk and the weights reduce-scattered
    in ascending rank order (the integer counts are exact either way)."""
    device = means3D.device
    empty = torch.empty(0, dtype=torch.float32, device=device)
    CH = int(image_weights.size(0))
    ws = pool.take(device)
    try:
        # this rank's means3D stands in the colors_precomp slot, as on one GPU: the colours are never used
        buf = shard_preprocess(plan, rs, means3D, empty, means3D, opacities, scales, rotations, cov3Ds_precomp, ws=ws)
        if buf.peer is not None:
            exchange.barrier(device)
        else:
            exchange.all_gather_inplace(exchange_view(buf))
        shard_order(buf)
        w_total = buf.alloc("aw_weights", plan.P_pad * CH, torch.float32, device).view(plan.P_pad, CH).zero_()
        c_total = buf.alloc("aw_cnt", plan.P_pad, torch.int32, device).zero_()
        shard_apply_weights(buf, image_weights, w_total, c_total, deterministic)
        w_slice = buf.alloc("aw_weights_slice", plan.slice_len * CH, torch.float32, device).view(plan.slice_len, CH)
        c_slice = buf.alloc("aw_cnt_slice", plan.slice_len, torch.int32, device)
        (exchange.reduce_scatter_ordered if deterministic else exchange.reduce_scatter_sum)(w_total, w_slice)
        exchange.reduce_scatter_sum(c_total, c_slice)
        n = plan.count
        weights.view(n, CH).add_(w_slice[:n])
        cnt.view(n).add_(c_slice[:n])
    finally:
        pool.give(ws)


# ---------------------------------------------------------------------------------------------------------
# autograd + module (one process per GPU)
# ---------------------------------------------------------------------------------------------------------
def grads_in_slots(grads, raw: bool):
    """The step functions' gradient tuple in the input slots of _ShardedRasterize / _SparseShardedRasterize:
    (means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp) and, last, features_rest. A raw
    shard has features_dc in the sh slot, the logits / log-scales / raw rotations in theirs and no colour or cov3D."""
    if raw:
        d_m3, d_m2, d_op, d_dc, d_rest, d_sc, d_ro = grads
        return (d_m3, d_m2, d_dc, None, d_op, d_sc, d_ro, None), d_rest
    return grads, None


class _ShardedRasterize(torch.autograd.Function):
    """Dense exchange. `raw_rest` (features_rest) makes it the fused-activation call (see shard_preprocess);
    `depth_grad` makes the depth output differentiable, with GaussianRasterizer(depth_grad=True)'s semantics;
    `return_alpha` adds the alpha output (a fifth frame plane); `viewmatrix` / `projmatrix` / `campos` (the settings'
    camera arrays, or None) are the camera inputs of camera_grad; `grad_mask` (uint8 [n] or None) selects the masked
    preprocess and backward."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, plan,
                exchange, pool, deterministic=False, depth_grad=False, raw_rest=None, return_alpha=False,
                viewmatrix=None, projmatrix=None, campos=None, grad_mask=None):
        ws = pool.take(means3D.device) if pool is not None else None
        buf = shard_preprocess(plan, rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                               ws=ws, raw_rest=raw_rest, grad_mask=grad_mask)
        if ws is not None:
            weakref.finalize(buf, pool.give, ws)     # back to the pool when the last user of this forward is gone
        if buf.peer is not None:
            exchange.barrier(means3D.device)           # every rank's records have landed everywhere
        else:
            exchange.all_gather_inplace(exchange_view(buf))
        shard_order(buf)
        frame = torch.zeros(5 if return_alpha else 4, buf.H, buf.W, dtype=torch.float32, device=means3D.device)
        shard_render(buf, frame[:3], frame[3:4])
        if return_alpha:
            shard_alpha(buf, frame[4:])
        exchange.all_reduce_sum(frame)
        ctx.buf, ctx.exchange, ctx.deterministic, ctx.depth_grad = buf, exchange, deterministic, bool(depth_grad)
        ctx.return_alpha, ctx.camera_grad, ctx.rs = bool(return_alpha), viewmatrix is not None, rs
        if ctx.depth_grad or ctx.return_alpha:
            # outputs without a gradient arrive as None: no depth / alpha gradient -> the ordinary backward, and a loss
            # on the depth or alpha alone leaves the colour gradient None (treated as zeros)
            ctx.set_materialize_grads(False)
        # a fresh tensor, like the single-GPU path and the reference: buf.radii lives in the pooled StepWorkspace and is
        # overwritten by the next forward that takes that workspace
        radii = shard_slice(buf.radii, plan).clone()
        ctx.mark_non_differentiable(radii)
        _ShardedRasterize.last_R = buf.R  # instrumentation only (no reference to the buffers: they must be free to die)
        if return_alpha:
            return frame[:3], radii, frame[3:4], frame[4:]
        return frame[:3], radii, frame[3:4]

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_alpha=None):
        buf, exchange, det = ctx.buf, ctx.exchange, ctx.deterministic
        grad_depth = grad_depth if ctx.depth_grad else None
        if grad_out_color is None:   # depth_grad / return_alpha: a loss on the depth or alpha alone
            grad_out_color = torch.zeros(3, buf.H, buf.W, dtype=torch.float32, device=buf.geom.device)
        acc = shard_backward_render(buf, grad_out_color, det, grad_depth, grad_alpha)
        acc_slice = buf.alloc("acc_slice", buf.plan.slice_len * ACC_STRIDE, torch.float32,
                              acc.device).view(buf.plan.slice_len, ACC_STRIDE)
        (exchange.reduce_scatter_ordered if det else exchange.reduce_scatter_sum)(acc, acc_slice)
        cam_grads = (None, None, None)
        if ctx.camera_grad:
            row, cam = camera_row(buf.plan.count, acc.device)
            grads = shard_backward_preprocess(buf, acc_slice, grad_depth is not None, cam)
            rows = torch.empty(exchange.world, CAM_ROW, dtype=torch.float32, device=acc.device)
            rows[exchange.rank].copy_(row)
            exchange.all_gather_inplace(rows)
            cam_grads = camera_grads_like(combine_camera_rows(rows), ctx.rs)
        else:
            grads = shard_backward_preprocess(buf, acc_slice, grad_depth is not None)
        grads, d_rest = grads_in_slots(grads, len(buf.inputs) == 8)
        return (*grads, None, None, None, None, None, None, d_rest, None, *cam_grads, None)


class _ShardedRasterizeStatic(torch.autograd.Function):
    """_ShardedRasterize for a fixed capacity (two more inputs, `capacity` and the device `status` int32[4]): no host
    copy and no host wait. The frame all-reduce carries one more float, this rank's overflow flag, and the gate empties
    the frame on every rank when any flag is set. The backward is _ShardedRasterize's, with R = capacity."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, plan,
                exchange, pool, deterministic=False, depth_grad=False, raw_rest=None, return_alpha=False,
                viewmatrix=None, projmatrix=None, campos=None, capacity=1, status=None, grad_mask=None):
        ws = pool.take(means3D.device)
        buf = shard_preprocess(plan, rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                               ws=ws, raw_rest=raw_rest, grad_mask=grad_mask)
        weakref.finalize(buf, pool.give, ws)
        buf.ws = StaticScratch(ws)                     # scratch of its own, never grown by apply_weights
        if buf.peer is not None:
            exchange.barrier(means3D.device)
        else:
            exchange.all_gather_inplace(exchange_view(buf))
        shard_order_static(buf, capacity)
        planes, npix = (5 if return_alpha else 4), buf.H * buf.W
        flat = torch.zeros(planes * npix + 1, dtype=torch.float32, device=means3D.device)
        frame = flat[:planes * npix].view(planes, buf.H, buf.W)
        shard_render_static(buf, frame[:3], frame[3:4], status)
        if return_alpha:
            shard_alpha(buf, frame[4:])
        flat[-1:].copy_(status[1:2])                   # this rank's 0/1 flag; the all-reduce sums it exactly
        exchange.all_reduce_sum(flat)
        static_gate(buf.s, buf.plan.P_pad, buf.geom, buf.img, frame, status, flag_sum=flat[-1:])
        ctx.buf, ctx.exchange, ctx.deterministic, ctx.depth_grad = buf, exchange, deterministic, bool(depth_grad)
        ctx.return_alpha, ctx.camera_grad, ctx.rs = bool(return_alpha), viewmatrix is not None, rs
        if ctx.depth_grad or ctx.return_alpha:
            ctx.set_materialize_grads(False)
        radii = shard_slice(buf.radii, plan).clone()
        ctx.mark_non_differentiable(radii)
        if return_alpha:
            return frame[:3], radii, frame[3:4], frame[4:]
        return frame[:3], radii, frame[3:4]

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_alpha=None):
        return (*_ShardedRasterize.backward(ctx, grad_out_color, grad_radii, grad_depth, grad_alpha), None, None)


def check_static_options(static_capacity, segment_capacity, mode: Optional[str], raster_settings):
    """The argument checks of ShardedGaussianRasterizer's fixed-capacity forward, made before any collective or device
    access. Returns (static_capacity, segment_capacity) as ints or None."""
    def as_count(v, name):   # GaussianRasterizer(static_capacity=...)'s check
        try:
            ok = not isinstance(v, bool) and int(v) == v and 0 < int(v) < 2 ** 31
        except (TypeError, ValueError):
            ok = False
        if not ok:
            raise ValueError(f"{name} must be an int in [1, 2^31), got {v!r}")
        return int(v)
    if static_capacity is None:
        if segment_capacity is not None:
            raise ValueError("segment_capacity needs static_capacity")
        return None, None
    static_capacity = as_count(static_capacity, "static_capacity")
    if segment_capacity is not None:
        segment_capacity = as_count(segment_capacity, "segment_capacity")
        if mode == "dense":
            raise ValueError("segment_capacity applies to mode='sparse' only")
    if raster_settings.debug:
        raise ValueError("static_capacity cannot be combined with debug=True: debug synchronises after every launch")
    return static_capacity, segment_capacity


def p2p_available(exchange: "Exchange") -> bool:
    """Peer mappings need every rank of the group on ONE node with peer access between all device pairs. Checked
    collectively (every rank gets the same answer), so that all ranks take the same code path."""
    import os
    if exchange.backend != "nccl" or exchange.world > 8:
        return False
    ok = int(os.environ.get("LOCAL_WORLD_SIZE", exchange.world)) == exchange.world
    try:
        me = torch.cuda.current_device()
        n = torch.cuda.device_count()
        ok = ok and n >= exchange.world and all(torch.cuda.can_device_access_peer(me, d) for d in range(n) if d != me)
    except Exception:
        ok = False
    flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=torch.device("cuda", torch.cuda.current_device()))
    exchange.dist.all_reduce(flag, op=exchange.dist.ReduceOp.MIN, group=exchange.group)
    return bool(int(flag[0]))


def check_sharded_grad_mask(mask, plan: ShardPlan, means3D, camera_grad: bool, raster_settings) -> torch.Tensor:
    """The checks of ``ShardedGaussianRasterizer.forward(..., grad_mask=...)``, made before any collective: this rank's
    rows [plan.count], bool or uint8, contiguous, on means3D's device; not with camera_grad. Returns the uint8 view."""
    if not isinstance(mask, torch.Tensor):
        raise ValueError(f"grad_mask must be a torch.Tensor, got {type(mask).__name__}")
    if mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"grad_mask must be a bool or uint8 tensor, got {mask.dtype}")
    if mask.dim() != 1 or mask.numel() != plan.count:
        raise ValueError(f"grad_mask must be this rank's rows [{plan.count}] (rank {plan.rank}), got shape "
                         f"{tuple(mask.shape)}")
    if not mask.is_contiguous():
        raise ValueError("grad_mask must be contiguous")
    if camera_grad:
        raise ValueError("grad_mask cannot be combined with camera_grad: the camera gradient sums over every Gaussian")
    if mask.device != means3D.device:
        raise ValueError(f"grad_mask is on {mask.device}, means3D on {means3D.device}")
    return mask.view(torch.uint8) if mask.dtype == torch.bool else mask


def check_forward_raw_flags(module):
    """forward_raw has neither the alpha output nor camera gradients (the fused-activation preprocess backward has no
    camera form, and the single-GPU forward_raw offers neither). Raised before any collective, so that the peers are
    not left waiting."""
    flags = [f for f in ("return_alpha", "camera_grad") if getattr(module, f, False)]
    if flags:
        raise ValueError(f"ShardedGaussianRasterizer.forward_raw is not available on a module built with "
                         f"{' and '.join(f + '=True' for f in flags)}: use forward with the activated parameters")


def _check_deterministic_flag():
    """By default the sharded backward and apply_weights add rows with float atomics, whose order changes from call to
    call. Under ``torch.use_deterministic_algorithms(True)`` that is an error (a warning with ``warn_only=True``), as for
    any PyTorch op without a deterministic implementation, unless the module was built with ``deterministic=True``."""
    if not torch.are_deterministic_algorithms_enabled():
        return
    msg = ("ShardedGaussianRasterizer(deterministic=None/False) is not deterministic: its backward and apply_weights add "
           "with float atomics. Construct it with deterministic=True (results reproducible for a fixed number of ranks), "
           "use the single-GPU GaussianRasterizer (deterministic mode) or turn the flag off with "
           "torch.use_deterministic_algorithms(False).")
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg)
    else:
        raise RuntimeError(msg)


class ShardedGaussianRasterizer(nn.Module):
    """``GaussianRasterizer`` for a cloud sharded by Gaussian index over the ranks of a process group.

    ``forward`` takes THIS RANK's rows of the per-Gaussian tensors (``shard_slice(full, plan)``) and returns the
    full image on every rank plus the radii of this rank's Gaussians; gradients flow to the local rows.

    ``mode``: ``"sparse"`` (default when peer mappings are available) -- records, the depth sort and the gradient rows
    only involve the ranks whose tile rows a Gaussian touches (sparse_sharded.py); ``"dense"`` -- every rank receives,
    sorts and reduces all P_total records (fused peer-store all-gather with ``p2p=True``, NCCL all-gather otherwise).
    ``max_in_flight``: forwards whose autograd state may be alive at the same time (GaussianEditor: 2; the peer-mapped
    workspaces are created collectively up front, one per slot).
    ``deterministic``: ``True`` selects the deterministic backward and ``apply_weights`` (no float atomics, partial
    sums of the ranks added in ascending rank order) in both modes and lets ``torch.use_deterministic_algorithms(True)``
    pass. Gradients, ``weights`` and ``cnt`` are then the same bits on every call and in every process for a FIXED
    number of ranks, and the dense and sparse modes give the same bits; at one rank they equal
    ``GaussianRasterizer(deterministic=True)``. With more ranks they are not the single-GPU bits (the sums are grouped
    per rank). ``None`` / ``False``: float atomics, and torch's deterministic flag raises (or warns).
    ``depth_grad``: ``True`` makes the depth output of ``forward`` and ``forward_raw`` differentiable, exactly as
    ``GaussianRasterizer(depth_grad=True)``: when the depth gets no gradient the ordinary backward runs, and a loss on
    the depth alone works (the colour gradient is then zeros). It combines with both modes and ``deterministic``.
    ``forward_raw`` is ``GaussianRasterizer.forward_raw`` (fused activations) on this rank's rows.
    ``return_alpha``: ``True`` makes ``forward`` return ``(color, radii_local, depth, alpha)``, alpha = 1 - final_T
    [1,H,W] (the full frame on every rank, bit-identical to ``GaussianRasterizer(return_alpha=True)``), differentiable.
    ``camera_grad``: ``True`` makes ``raster_settings.viewmatrix / projmatrix / campos`` autograd inputs, as on one GPU;
    their ``.grad`` on every rank is the gradient of the whole cloud (the ranks' partials added in ascending rank
    order), the same bits on every rank. Both combine with both modes, ``deterministic`` and ``depth_grad``; neither is
    available on ``forward_raw``.
    ``static_capacity`` (opt-in, an int in [1, 2^31)): ``GaussianRasterizer(static_capacity=N)`` for a sharded cloud. N
    is the instance capacity of this rank's owned tiles; ``forward`` and ``forward_raw`` (forward and backward) then never
    wait for the device and never touch host memory, so a sharded training step can be captured with
    ``torch.cuda.graph``. ``segment_capacity`` (sparse mode only; default: the allocation, which can never overflow) is
    the fixed capacity of every sparse segment, the records one rank sends to another. ``self.status`` is a device
    int32[4] ``{R of this rank, overflow, largest segment (sparse), barrier error (sparse)}``; overflow is 1 on EVERY rank
    when any rank's R exceeded N or any segment exceeded ``segment_capacity``, and that frame is then EMPTY on every rank
    (background colour, depth and alpha 0, every gradient exactly zero). Nothing checks it implicitly:
    ``check_capacity()`` synchronises and raises. Otherwise frames, radii and alpha are the default path's bits and
    gradients agree with it (bit for bit with ``deterministic=True``). ``apply_weights`` keeps its exact, host-sized path.
    Not combinable with ``raster_settings.debug``.
    ``grad_mask`` (opt-in, a per-call argument of ``forward`` and ``forward_raw``, not a constructor option: the mask
    changes whenever the cloud is densified): THIS RANK's rows [n] of ``GaussianRasterizer``'s ``grad_mask``, a bool
    (viewed as uint8, not copied) or uint8 CUDA tensor, contiguous. Only the Gaussians with ``grad_mask[i] != 0`` take
    gradients; every gradient row of the others is +0.0. The edit bit travels to the tile owners inside the splat
    records, whose exchange already exists, and their blend backward skips the unedited splats' work. Frames, radii,
    depth and alpha are unchanged; the edited rows equal the unmasked backward's (bit for bit with
    ``deterministic=True``). It is part of the collective contract: every rank passes a mask, or none does, exactly as
    every rank renders the same camera. The mask must hold the same values at the backward as at the forward (the blend
    backward uses the forward's bits, the preprocess backward reads the mask). It combines with both modes,
    ``deterministic``, ``depth_grad``, ``return_alpha`` and ``static_capacity`` (captured in a CUDA graph, the mask's
    storage is fixed and its contents may change between replays); not with ``camera_grad`` (ValueError).
    """

    def __init__(self, raster_settings: GaussianRasterizationSettings, P_total: int, group=None,
                 p2p: Optional[bool] = None, mode: Optional[str] = None, max_in_flight: int = 3,
                 deterministic: Optional[bool] = None, depth_grad: bool = False, return_alpha: bool = False,
                 camera_grad: bool = False, static_capacity=None, segment_capacity=None):
        super().__init__()
        self.raster_settings = raster_settings
        self.deterministic = bool(deterministic)
        self.depth_grad = bool(depth_grad)
        self.return_alpha = bool(return_alpha)
        self.camera_grad = bool(camera_grad)
        # checked before any collective: a bad option raises on its rank instead of leaving the peers waiting
        self.static_capacity, self.segment_capacity = check_static_options(static_capacity, segment_capacity, mode,
                                                                           raster_settings)
        self.status = None   # device int32[4] of the last static forward
        self.exchange = Exchange(group)
        self.plan = ShardPlan(int(P_total), self.exchange.world, self.exchange.rank)
        if self.segment_capacity is not None and self.segment_capacity > max(self.plan.slice_len, 1):
            raise ValueError(f"segment_capacity must be in [1, {max(self.plan.slice_len, 1)}] (the allocation), got "
                             f"{self.segment_capacity}")
        can_p2p = p2p_available(self.exchange) if (p2p is None or p2p or mode == "sparse") else False
        if p2p and not can_p2p:
            raise RuntimeError("p2p=True needs all ranks on one node with peer access between every device pair")
        if mode is None:
            mode = "sparse" if (can_p2p and p2p is not False) else "dense"
        if mode not in ("sparse", "dense"):
            raise ValueError("mode must be 'sparse' or 'dense'")
        if mode == "sparse" and not can_p2p:
            raise RuntimeError("mode='sparse' needs peer mappings (all ranks on one node with peer access)")
        if mode == "dense" and self.segment_capacity is not None:   # (mode=None resolved to dense: same on every rank)
            raise ValueError("segment_capacity applies to mode='sparse' only")
        self.mode = mode
        self.pool = self.sparse_pool = None
        if mode == "sparse":
            from . import sparse_sharded as SS
            dev = torch.device("cuda", torch.cuda.current_device())
            self.sparse_pool = SS.SparsePool(self.plan, dev, int(raster_settings.image_width),
                                             int(raster_settings.image_height), self.exchange, depth=max_in_flight,
                                             alpha=self.return_alpha, camera=self.camera_grad,
                                             device_epoch=self.static_capacity is not None)
        else:
            # fused preprocess + all-gather through peer-mapped workspaces (faster than the NCCL all-gather)
            self.pool = WorkspacePool(self.exchange, _geometry_bytes(_lib.load(), self.plan.P_pad),
                                      bool(can_p2p if p2p is None else p2p))

    def close(self):
        """Release the peer-mapped and step workspaces (collective: every rank must call it). A densified cloud gets a
        new module: ``close()`` and construct ``ShardedGaussianRasterizer(rs, P_new, ...)``, as often as needed in one
        process group. Calling ``close()`` again does nothing; a closed module cannot render."""
        if self.pool is not None:
            self.pool.close()
        if self.sparse_pool is not None:
            self.sparse_pool.close()
        self.pool = self.sparse_pool = None
        self.closed = True

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, grad_mask=None):
        if grad_mask is not None:
            grad_mask = check_sharded_grad_mask(grad_mask, self.plan, means3D, self.camera_grad, self.raster_settings)
        if not getattr(self, "deterministic", False):
            _check_deterministic_flag()
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or (
                (scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        empty = torch.empty(0, dtype=torch.float32, device=means3D.device)
        shs = empty if shs is None else shs
        colors_precomp = empty if colors_precomp is None else colors_precomp
        scales = empty if scales is None else scales
        rotations = empty if rotations is None else rotations
        cov3D_precomp = empty if cov3D_precomp is None else cov3D_precomp
        return self._apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, None,
                           grad_mask)

    def forward_raw(self, means3D, means2D, opacity_logits, features_dc, features_rest, log_scales, raw_rotations,
                    grad_mask=None):
        """``GaussianRasterizer.forward_raw`` of a sharded cloud (collective): THIS RANK's rows of the scene model's raw
        parameters (``_xyz, _opacity, _features_dc, _features_rest, _scaling, _rotation``); the activations and the SH
        concatenation happen inside the preprocess kernels. Returns ``(color, radii_local, depth)`` as ``forward``;
        gradients land on the raw local leaves (``means2D`` included). ``grad_mask``: as in ``forward``."""
        check_forward_raw_flags(self)
        if grad_mask is not None:
            grad_mask = check_sharded_grad_mask(grad_mask, self.plan, means3D, self.camera_grad, self.raster_settings)
        if not getattr(self, "deterministic", False):
            _check_deterministic_flag()
        if means3D.dim() != 2 or means3D.size(1) != 3:
            raise RuntimeError("means3D must have dimensions (num_points, 3)")
        empty = torch.empty(0, dtype=torch.float32, device=means3D.device)
        return self._apply(means3D, means2D, features_dc, empty, opacity_logits, log_scales, raw_rotations, empty,
                           features_rest, grad_mask)

    def _apply(self, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3D_precomp, raw_rest,
               grad_mask=None):
        if getattr(self, "closed", False):
            raise RuntimeError("this ShardedGaussianRasterizer was closed: construct a new one")
        rs = self.raster_settings
        depth_grad = getattr(self, "depth_grad", False)
        return_alpha = getattr(self, "return_alpha", False)
        cam = (rs.viewmatrix, rs.projmatrix, rs.campos) if getattr(self, "camera_grad", False) else (None, None, None)
        if getattr(self, "static_capacity", None) is not None:
            return self._apply_static(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3D_precomp,
                                      raw_rest, depth_grad, return_alpha, cam, grad_mask)
        if self.mode == "sparse":
            from . import sparse_sharded as SS
            rk0 = self.sparse_pool.all[0]
            if int(rs.image_width) != rk0.W or int(rs.image_height) != rk0.H:
                raise RuntimeError("sparse mode: the image size is fixed at construction (peer-mapped frames)")
            return SS._SparseShardedRasterize.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                                    cov3D_precomp, rs, self.sparse_pool, self.exchange,
                                                    self.deterministic, depth_grad, raw_rest, return_alpha, *cam,
                                                    grad_mask)
        return _ShardedRasterize.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                       cov3D_precomp, rs, self.plan, self.exchange, self.pool, self.deterministic,
                                       depth_grad, raw_rest, return_alpha, *cam, grad_mask)

    def _apply_static(self, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3D_precomp, raw_rest,
                      depth_grad, return_alpha, cam, grad_mask=None):
        rs = self.raster_settings
        if rs.debug:
            raise ValueError("static_capacity cannot be combined with debug=True: debug synchronises after every launch")
        if self.status is None or self.status.device != means3D.device:
            self.status = torch.zeros(STATUS_WORDS, dtype=torch.int32, device=means3D.device)
        if self.mode == "sparse":
            from . import sparse_sharded as SS
            rk0 = self.sparse_pool.all[0]
            if int(rs.image_width) != rk0.W or int(rs.image_height) != rk0.H:
                raise RuntimeError("sparse mode: the image size is fixed at construction (peer-mapped frames)")
            seg_cap = self.segment_capacity if self.segment_capacity is not None else rk0.cap_alloc
            return SS._SparseShardedRasterizeStatic.apply(
                means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3D_precomp, rs, self.sparse_pool,
                self.exchange, self.deterministic, depth_grad, raw_rest, return_alpha, *cam, self.static_capacity,
                seg_cap, self.status, grad_mask)
        return _ShardedRasterizeStatic.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                             cov3D_precomp, rs, self.plan, self.exchange, self.pool, self.deterministic,
                                             depth_grad, raw_rest, return_alpha, *cam, self.static_capacity,
                                             self.status, grad_mask)

    def check_capacity(self) -> int:
        """Synchronise with the last static forward and raise RuntimeError if it overflowed anywhere (that frame was
        rendered empty on every rank) or a peer barrier timed out. The answer is the same on every rank; the message
        names what overflowed. Returns this rank's instance count R otherwise. Never called implicitly."""
        if self.static_capacity is None or self.status is None:
            raise RuntimeError("check_capacity() needs a static_capacity rasterizer that has run a forward")
        seg = None
        if self.mode == "sparse":
            seg = self.segment_capacity if self.segment_capacity is not None else self.sparse_pool.all[0].cap_alloc
        status = self.status.cpu()
        msg = static_status_error(status, self.static_capacity, seg, self.plan.rank)
        if msg is not None:
            raise RuntimeError(msg)
        return int(status[0])

    def apply_weights(self, means3D, means2D, opacities, shs=None, weights=None, scales=None, rotations=None,
                      cov3Ds_precomp=None, cnt=None, image_weights=None):
        """Semantic tracing of the sharded cloud (``GaussianRasterizer.apply_weights``, collective: every rank calls it
        for the same view). The per-Gaussian tensors, ``weights`` [n,CH] float32 and ``cnt`` [n,1] int32 are THIS RANK's
        rows and are updated in place (accumulated over calls); ``image_weights`` [CH,H,W] is the full mask, the same on
        every rank. ``cnt`` equals the single-GPU result bit for bit, ``weights`` up to the order of the float sums
        (bit for bit from call to call with ``deterministic=True``)."""
        if getattr(self, "closed", False):
            raise RuntimeError("this ShardedGaussianRasterizer was closed: construct a new one")
        if not getattr(self, "deterministic", False):
            _check_deterministic_flag()
        rs = self.raster_settings
        check_apply_weights_args(self.plan, rs, means3D, weights, cnt, image_weights, scales, rotations, cov3Ds_precomp)
        empty = torch.empty(0, dtype=torch.float32, device=means3D.device)
        scales = empty if scales is None else scales
        rotations = empty if rotations is None else rotations
        cov3Ds_precomp = empty if cov3Ds_precomp is None else cov3Ds_precomp
        with torch.no_grad():
            if self.mode == "sparse":
                from . import sparse_sharded as SS
                SS.sparse_apply_weights(self.sparse_pool, rs, means3D, opacities, scales, rotations, cov3Ds_precomp,
                                        image_weights, weights, cnt, self.deterministic)
            else:
                dense_apply_weights(self.plan, self.exchange, self.pool, rs, means3D, opacities, scales, rotations,
                                    cov3Ds_precomp, image_weights, weights, cnt, self.deterministic)

    def markVisible(self, positions):
        """``GaussianRasterizer.markVisible`` of this rank's rows ``positions`` [n,3] (no collective)."""
        return mark_visible(self.raster_settings, positions)
