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
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib
from .rasterizer import (GaussianRasterizationSettings, _f32c, _geometry_bytes, _make_cloud, _make_settings,
                         _pinned_i32, _ptr)

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

    def reduce_scatter_sum(self, total: torch.Tensor, out: torch.Tensor):
        """out[n, ...] = sum over ranks of total[rank*n:(rank+1)*n]."""
        if self.backend == "nccl":
            self.dist.reduce_scatter_tensor(out, total, op=self.dist.ReduceOp.SUM, group=self.group)
        else:  # gloo: no reduce-scatter
            tmp = total.clone()
            self.dist.all_reduce(tmp, op=self.dist.ReduceOp.SUM, group=self.group)
            n = out.shape[0]
            out.copy_(tmp[self.rank * n:(self.rank + 1) * n])


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
                 "ws", "__weakref__")

    def alloc(self, name: str, numel: int, dtype, device, grow: float = 1.0) -> torch.Tensor:
        """A scratch buffer: from the persistent StepWorkspace when there is one, else from the caching allocator."""
        if self.ws is not None:
            return self.ws.get(name, numel, dtype, grow)
        return torch.empty(numel, dtype=dtype, device=device)


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
                     ws: Optional[StepWorkspace] = None) -> ShardBuffers:
    """Stage 1: project this rank's Gaussians into its slice of the global arrays. `geom` / `radii` may be passed
    in to share one set of global arrays between virtual ranks of a single process. With `peer` (a PeerWorkspace of
    gsr_geometry_bytes(P_pad) bytes) the kernel pushes its records into every rank's workspace itself: no all-gather
    follows, only a barrier. `ws` (a StepWorkspace) supplies all scratch buffers persistently, its `peer` included."""
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
    buf = ShardBuffers()
    buf.plan, buf.M, buf.W, buf.H, buf.ws = plan, M, W, H, ws
    with torch.cuda.device(device):
        means3D = _f32c(means3D, device); opacities = _f32c(opacities, device)
        sh = _f32c(sh, device); colors_precomp = _f32c(colors_precomp, device)
        scales = _f32c(scales, device); rotations = _f32c(rotations, device)
        cov3Ds_precomp = _f32c(cov3Ds_precomp, device)
        buf.inputs = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
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
        c = _make_cloud(plan.count, means3D, opacities, sh, colors_precomp, scales, rotations, cov3Ds_precomp)
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        if peer is not None:
            _lib.check(lib.gsr_shard_preprocess_p2p(C.byref(s), C.byref(c), plan.P_pad, plan.base, plan.slice_len,
                                                    peer.ptr_array, plan.world, plan.rank, peer.nbytes,
                                                    _ptr(buf.radii), st), "gsr_shard_preprocess_p2p")
        else:
            _lib.check(lib.gsr_shard_preprocess(C.byref(s), C.byref(c), plan.P_pad, plan.base, plan.slice_len,
                                                _ptr(buf.geom), gbytes, _ptr(buf.radii), st), "gsr_shard_preprocess")
    return buf


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


def shard_backward_render(buf: ShardBuffers, grad_out_color: torch.Tensor) -> torch.Tensor:
    """Backward stage 1: this rank's tiles -> partial accumulators [P_pad, 12] (zero for untouched Gaussians)."""
    lib = _lib.load()
    device = buf.geom.device
    with torch.cuda.device(device):
        s, own = buf.s, buf.own
        grad_out_color = _f32c(grad_out_color, device)
        acc = buf.alloc("acc", buf.plan.P_pad * ACC_STRIDE, torch.float32, device).view(buf.plan.P_pad, ACC_STRIDE)
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(lib.gsr_shard_backward_render(C.byref(s), C.byref(own), buf.plan.P_pad, buf.R, _ptr(buf.geom),
                                                 buf.geom.numel(), _ptr(buf.binning), buf.binning.numel(),
                                                 _ptr(buf.img), buf.img.numel(), _ptr(grad_out_color), _ptr(acc),
                                                 acc.numel() * 4, st), "gsr_shard_backward_render")
    return acc


def shard_backward_preprocess(buf: ShardBuffers, acc_slice: torch.Tensor):
    """Backward stage 2 (after the reduce-scatter): gradients of this rank's Gaussians, reference slot order."""
    lib = _lib.load()
    device = buf.geom.device
    plan, M = buf.plan, buf.M
    n = plan.count
    (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp) = buf.inputs
    with torch.cuda.device(device):
        f32 = dict(dtype=torch.float32, device=device)
        dL_dmeans3D = torch.empty(n, 3, **f32); dL_dmeans2D = torch.empty(n, 3, **f32)
        dL_dcolors = torch.empty(n, 3, **f32); dL_dopacity = torch.empty(n, 1, **f32)
        dL_dcov3D = torch.empty(n, 6, **f32); dL_dsh = torch.empty(n, M, 3, **f32)
        dL_dscales = torch.empty(n, 3, **f32); dL_drotations = torch.empty(n, 4, **f32)
        if n > 0:
            s = buf.s
            c = _make_cloud(n, means3D, opacities, sh, colors_precomp, scales, rotations, cov3Ds_precomp)
            gr = _lib.Grads(_ptr(dL_dmeans3D), _ptr(dL_dmeans2D), _ptr(dL_dcolors), _ptr(dL_dopacity),
                            _ptr(dL_dcov3D), _ptr(dL_dsh), _ptr(dL_dscales), _ptr(dL_drotations))
            st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
            _lib.check(lib.gsr_shard_backward_preprocess(C.byref(s), C.byref(c), plan.P_pad, plan.base, _ptr(buf.geom),
                                                         buf.geom.numel(), _ptr(buf.radii), _ptr(acc_slice),
                                                         C.byref(gr), st), "gsr_shard_backward_preprocess")
            if scales.numel() == 0:
                dL_dscales.zero_(); dL_drotations.zero_()
    return (dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D)


# ---------------------------------------------------------------------------------------------------------
# autograd + module (one process per GPU)
# ---------------------------------------------------------------------------------------------------------
class _ShardedRasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, plan,
                exchange, pool):
        ws = pool.take(means3D.device) if pool is not None else None
        buf = shard_preprocess(plan, rs, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                               ws=ws)
        if ws is not None:
            weakref.finalize(buf, pool.give, ws)     # back to the pool when the last user of this forward is gone
        if buf.peer is not None:
            exchange.barrier(means3D.device)           # every rank's records have landed everywhere
        else:
            exchange.all_gather_inplace(exchange_view(buf))
        shard_order(buf)
        frame = torch.zeros(4, buf.H, buf.W, dtype=torch.float32, device=means3D.device)
        shard_render(buf, frame[:3], frame[3:])
        exchange.all_reduce_sum(frame)
        ctx.buf, ctx.exchange = buf, exchange
        # a fresh tensor, like the single-GPU path and the reference: buf.radii lives in the pooled StepWorkspace and is
        # overwritten by the next forward that takes that workspace
        radii = shard_slice(buf.radii, plan).clone()
        ctx.mark_non_differentiable(radii)
        _ShardedRasterize.last_R = buf.R  # instrumentation only (no reference to the buffers: they must be free to die)
        return frame[:3], radii, frame[3:]

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth):
        buf, exchange = ctx.buf, ctx.exchange
        acc = shard_backward_render(buf, grad_out_color)
        acc_slice = buf.alloc("acc_slice", buf.plan.slice_len * ACC_STRIDE, torch.float32,
                              acc.device).view(buf.plan.slice_len, ACC_STRIDE)
        exchange.reduce_scatter_sum(acc, acc_slice)
        grads = shard_backward_preprocess(buf, acc_slice)
        return (*grads, None, None, None, None)


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


class ShardedGaussianRasterizer(nn.Module):
    """``GaussianRasterizer`` for a cloud sharded by Gaussian index over the ranks of a process group.

    ``forward`` takes THIS RANK's rows of the per-Gaussian tensors (``shard_slice(full, plan)``) and returns the
    full image on every rank plus the radii of this rank's Gaussians; gradients flow to the local rows.

    ``mode``: ``"sparse"`` (default when peer mappings are available) -- records, the depth sort and the gradient rows
    only involve the ranks whose tile rows a Gaussian touches (sparse_sharded.py); ``"dense"`` -- every rank receives,
    sorts and reduces all P_total records (fused peer-store all-gather with ``p2p=True``, NCCL all-gather otherwise).
    ``max_in_flight``: forwards whose autograd state may be alive at the same time (GaussianEditor: 2; the peer-mapped
    workspaces are created collectively up front, one per slot).
    """

    def __init__(self, raster_settings: GaussianRasterizationSettings, P_total: int, group=None,
                 p2p: Optional[bool] = None, mode: Optional[str] = None, max_in_flight: int = 3):
        super().__init__()
        self.raster_settings = raster_settings
        self.exchange = Exchange(group)
        self.plan = ShardPlan(int(P_total), self.exchange.world, self.exchange.rank)
        can_p2p = p2p_available(self.exchange) if (p2p is None or p2p or mode == "sparse") else False
        if p2p and not can_p2p:
            raise RuntimeError("p2p=True needs all ranks on one node with peer access between every device pair")
        if mode is None:
            mode = "sparse" if (can_p2p and p2p is not False) else "dense"
        if mode not in ("sparse", "dense"):
            raise ValueError("mode must be 'sparse' or 'dense'")
        if mode == "sparse" and not can_p2p:
            raise RuntimeError("mode='sparse' needs peer mappings (all ranks on one node with peer access)")
        self.mode = mode
        self.pool = self.sparse_pool = None
        if mode == "sparse":
            from . import sparse_sharded as SS
            dev = torch.device("cuda", torch.cuda.current_device())
            self.sparse_pool = SS.SparsePool(self.plan, dev, int(raster_settings.image_width),
                                             int(raster_settings.image_height), self.exchange, depth=max_in_flight)
        else:
            # fused preprocess + all-gather through peer-mapped workspaces (faster than the NCCL all-gather)
            self.pool = WorkspacePool(self.exchange, _geometry_bytes(_lib.load(), self.plan.P_pad),
                                      bool(can_p2p if p2p is None else p2p))

    def close(self):
        """Release the peer-mapped workspaces (collective: every rank must call it)."""
        if self.pool is not None:
            self.pool.close()
        if self.sparse_pool is not None:
            self.sparse_pool.close()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
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
        rs = self.raster_settings
        if self.mode == "sparse":
            from . import sparse_sharded as SS
            rk0 = self.sparse_pool.all[0]
            if int(rs.image_width) != rk0.W or int(rs.image_height) != rk0.H:
                raise RuntimeError("sparse mode: the image size is fixed at construction (peer-mapped frames)")
            return SS._SparseShardedRasterize.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                                    cov3D_precomp, rs, self.sparse_pool, self.exchange)
        return _ShardedRasterize.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                       cov3D_precomp, rs, self.plan, self.exchange, self.pool)
