"""Drop-in replacement of the reference's ``diff_gaussian_rasterization`` Python package.

Same public names, argument meaning, return values and error messages as
/root/reference/gaussiansplatting/submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py
(``GaussianRasterizationSettings`` :228-240, ``GaussianRasterizer`` :243-364, ``rasterize_gaussians`` :26-47,
``_RasterizeGaussians`` :50-225), backed by the sm_90a C-ABI library instead of the ``_C`` pybind module.

Differences a caller can observe (all documented in DESIGN.md):
  * kernels run on PyTorch's CURRENT stream (the reference always used the legacy default stream);
  * the only host synchronisation per forward is one stream sync to read ``num_rendered``, and none at all with
    ``static_capacity`` (the forward then only enqueues work, so a whole training step can be captured in a CUDA graph);
  * gradient tensors are written completely by the kernels (no separate zero-fill passes);
  * ``debug=True`` synchronises after every launch and raises on the first CUDA error, but does not write the
    reference's ``snapshot_*.dump`` files.
"""
from __future__ import annotations

import ctypes as C
import threading
import time
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _lib


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


_size_cache: dict = {}
_pinned: dict = {}
_r_hint: dict = {}          # (device, P, W, H) -> largest num_rendered seen recently
SPECULATIVE = True          # launch the second forward half before num_rendered is known (see _forward_impl)
SPEC_STATS = {"launched": 0, "missed": 0}   # speculative second halves launched / redone because the guess was too small


def _f32c(t: torch.Tensor, device) -> torch.Tensor:
    """float32, contiguous, on `device`, 16-byte aligned storage."""
    if t.dtype != torch.float32 or t.device != device or not t.is_contiguous():
        t = t.to(device=device, dtype=torch.float32).contiguous()
    if t.data_ptr() % 16:
        t = t.clone()
    return t


def _ptr(t):
    return None if t is None or t.numel() == 0 else C.c_void_p(t.data_ptr())


def _bounded_put(d: dict, key, value, limit: int = 64):
    """Densification changes P every few hundred steps: keep the per-(P, W, H) dictionaries from growing forever."""
    if key not in d and len(d) >= limit:
        d.pop(next(iter(d)))
    d[key] = value


def _geometry_bytes(lib, P):
    key = ("g", P)
    if key not in _size_cache:
        n = lib.gsr_geometry_bytes(P)
        if n == 0:
            _lib.check(-2, "gsr_geometry_bytes")
        _bounded_put(_size_cache, key, n)
    return _size_cache[key]


def _pinned_i32(device):
    """One pinned count word per (device, stream, host thread): two threads driving forwards on the same stream (e.g. the
    autograd engine thread re-running a checkpointed forward) must not poll each other's word."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream, threading.get_ident())
    if key not in _pinned:
        _bounded_put(_pinned, key, torch.zeros(1, dtype=torch.int32).pin_memory(), limit=256)
    return _pinned[key]


def _wait_count(pinned: torch.Tensor, waiter) -> int:
    """num_rendered arrives in a pinned host word (preset to -1) through an async copy that the library issues right
    behind the preprocess kernel, i.e. BEFORE the depth sort it has already queued: spinning on the word hands the
    count to the host while the GPU is still busy, instead of sleeping until the whole first half has drained.
    Falls back to `waiter()` (event / stream synchronize) after 2 ms."""
    t0 = time.perf_counter()
    while int(pinned[0]) < 0:
        if time.perf_counter() - t0 > 2e-3:
            waiter()
            break
    return int(pinned[0])


def _make_settings(rs: GaussianRasterizationSettings, M: int, device, keep: list) -> _lib.Settings:
    bg = _f32c(rs.bg, device); view = _f32c(rs.viewmatrix, device)
    proj = _f32c(rs.projmatrix, device); campos = _f32c(rs.campos, device)
    keep += [bg, view, proj, campos]
    return _lib.Settings(int(rs.image_height), int(rs.image_width), float(rs.tanfovx), float(rs.tanfovy),
                         float(rs.scale_modifier), int(rs.sh_degree), int(M), int(bool(rs.prefiltered)),
                         int(bool(rs.debug)), bg.data_ptr(), view.data_ptr(), proj.data_ptr(), campos.data_ptr())


def _make_cloud(P, means3D, opacities, sh, colors_precomp, scales, rotations, cov3Ds_precomp) -> _lib.Cloud:
    return _lib.Cloud(P, _ptr(means3D), _ptr(opacities), _ptr(sh), _ptr(colors_precomp), _ptr(scales),
                      _ptr(rotations), _ptr(cov3Ds_precomp))


class _ForwardState:
    """What the forward leaves behind for backward / apply_weights / parity tests."""
    __slots__ = ("geom", "binning", "img", "radii", "num_rendered", "cap", "P", "M", "W", "H", "mask_first")


def _mask_twin(lib, name, mask_render, keep):
    """(entry point, its name, trailing arguments before the stream): ``name`` itself, or with ``mask_render = (mask,
    out)`` its _mask twin, which also writes the mask image into ``out`` [3,H,W]. The twins take no NULL pointer, so an
    empty mask (P = 0) or image (W*H = 0) is handed over as a one-element buffer that is never read or written."""
    if mask_render is None:
        return getattr(lib, name), name, ()
    ptrs = []
    for t in mask_render:
        if t.numel() == 0:
            t = torch.zeros(1, dtype=t.dtype, device=t.device)
        keep.append(t)
        ptrs.append(C.c_void_p(t.data_ptr()))
    return getattr(lib, name + "_mask"), name + "_mask", tuple(ptrs)


def _forward_impl(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, *, render=True,
                  raw_rest=None, static=None, mask_render=None):
    """Both forward halves. With ``raw_rest`` (features_rest [P,K,3]) the call is the fused-activation variant:
    ``sh`` is features_dc [P,1,3] and opacities / scales / rotations are the raw parameters.
    With ``static = (capacity, status)`` both halves run in one gsr_forward_static call sized for ``capacity``: no
    pinned word, no host wait; num_rendered and the overflow flag land in the device tensor ``status`` int32[2].
    With ``mask_render = (mask, out)`` (uint8 [P], float32 [3,H,W]) the second half also writes the mask image into
    ``out`` (the _mask twin of each forward entry point)."""
    lib = _lib.load()
    if means3D.dim() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:46-48
    if not means3D.is_cuda:
        raise RuntimeError("the rasterizer needs CUDA tensors (there is no CPU path)")
    device = means3D.device
    P = means3D.size(0)
    H, W = int(rs.image_height), int(rs.image_width)
    M = sh.size(1) if sh.dim() >= 2 else 0   # from the shape: an empty cloud's dL/dsh is [0, M, 3] like its input
    raw = raw_rest is not None
    if raw:
        M = 1 + raw_rest.size(1)
    with torch.cuda.device(device):
        if raw:
            raw_rest = _f32c(raw_rest, device)
        means3D = _f32c(means3D, device); opacities = _f32c(opacities, device)
        sh = _f32c(sh, device); colors_precomp = _f32c(colors_precomp, device)
        scales = _f32c(scales, device); rotations = _f32c(rotations, device)
        cov3Ds_precomp = _f32c(cov3Ds_precomp, device)
        keep = []
        s = _make_settings(rs, M, device, keep)
        c = _make_cloud(P, means3D, opacities, sh, colors_precomp, scales, rotations, cov3Ds_precomp)
        stream = torch.cuda.current_stream(device)
        st = C.c_void_p(stream.cuda_stream)
        u8 = dict(dtype=torch.uint8, device=device)
        state = _ForwardState()
        state.P, state.M, state.W, state.H = P, M, W, H
        state.radii = torch.empty(P, dtype=torch.int32, device=device)
        gbytes = _geometry_bytes(lib, P) if P > 0 else 0
        state.geom = torch.empty(gbytes, **u8)
        if static is not None:
            cap, status = static
            color, depth = _forward_static(lib, s, c, P, W, H, cap, status, gbytes, state, st, device,
                                           raw_rest if raw else None, mask_render)
            inputs = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
            return color, depth, state, inputs + ((raw_rest,) if raw else ())
        pinned = _pinned_i32(device)
        pinned[0] = -1
        if raw:
            rc = _lib.RawCloud(P, _ptr(means3D), _ptr(opacities), _ptr(sh), _ptr(raw_rest), _ptr(scales), _ptr(rotations))
            _lib.check(lib.gsr_forward_preprocess_raw(C.byref(s), C.byref(rc), _ptr(state.geom), gbytes,
                                                      _ptr(state.radii), C.c_void_p(pinned.data_ptr()), st),
                       "gsr_forward_preprocess_raw")
        else:
            _lib.check(lib.gsr_forward_preprocess(C.byref(s), C.byref(c), _ptr(state.geom), gbytes, _ptr(state.radii),
                                                  C.c_void_p(pinned.data_ptr()), st), "gsr_forward_preprocess")
        ibytes = lib.gsr_image_bytes(W, H)
        state.img = torch.empty(ibytes, **u8)
        color = depth = None
        if render:
            color = torch.empty(3, H, W, dtype=torch.float32, device=device)
            depth = torch.empty(1, H, W, dtype=torch.float32, device=device)
        key = (device.index, P, W, H)
        hint = _r_hint.get(key)
        done = False
        if SPECULATIVE and render and P > 0 and hint:
            # The count of (Gaussian, tile) instances is only known on the device at this point. Instead of idling
            # the GPU while the host fetches it (the reference blocks in cudaMemcpy), enqueue the second half now for
            # a guessed capacity, THEN wait for the count: the GPU keeps working while the host waits. A wrong guess
            # (count > capacity) is detected below and the second half is redone with the exact size.
            ev = torch.cuda.Event()
            ev.record(stream)
            cap = int(hint * 1.25) + 4096
            bbytes = lib.gsr_binning_bytes(P, cap, W, H)
            state.binning = torch.empty(bbytes, **u8)
            fn, name, mr = _mask_twin(lib, "gsr_forward_render_speculative", mask_render, keep)
            _lib.check(fn(C.byref(s), C.byref(c), cap, _ptr(state.geom), gbytes, _ptr(state.binning), bbytes,
                          _ptr(state.img), ibytes, _ptr(state.radii), _ptr(color), _ptr(depth), *mr, st), name)
            R = _wait_count(pinned, ev.synchronize)
            SPEC_STATS["launched"] += 1
            if R <= cap:
                state.num_rendered, state.cap, done = R, cap, True
            else:
                SPEC_STATS["missed"] += 1
        if not done:
            R = _wait_count(pinned, stream.synchronize)
            state.num_rendered = state.cap = R
            bbytes = lib.gsr_binning_bytes(P, R, W, H) if R > 0 else 0
            state.binning = torch.empty(bbytes, **u8)
            if render:
                fn, name, mr = _mask_twin(lib, "gsr_forward_render", mask_render, keep)
                _lib.check(fn(C.byref(s), C.byref(c), R, _ptr(state.geom), gbytes, _ptr(state.binning), bbytes,
                              _ptr(state.img), ibytes, _ptr(state.radii), _ptr(color), _ptr(depth), *mr, st), name)
        if P > 0:
            _bounded_put(_r_hint, key, max(R, int(0.9 * _r_hint.get(key, 0))))
    inputs = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
    if raw:
        inputs = inputs + (raw_rest,)
    return color, depth, state, inputs


def _forward_static(lib, s, c, P, W, H, cap, status, gbytes, state, st, device, raw_rest, mask_render=None):
    """Second half of _forward_impl on the static-capacity path (gsr_forward_static / gsr_forward_static_raw).
    Returns (colour, depth); the state keeps no reference to them (the autograd node holds the state)."""
    u8 = dict(dtype=torch.uint8, device=device)
    bbytes = lib.gsr_binning_bytes(P, cap, W, H)
    if bbytes == 0:
        _lib.check(-2, "gsr_binning_bytes")
    state.binning = torch.empty(bbytes, **u8)
    ibytes = lib.gsr_image_bytes(W, H)
    state.img = torch.empty(ibytes, **u8)
    color = torch.empty(3, H, W, dtype=torch.float32, device=device)
    depth = torch.empty(1, H, W, dtype=torch.float32, device=device)
    state.num_rendered, state.cap = None, cap   # R is on the device only (status[0])
    keep = []
    fn, name, mr = _mask_twin(lib, "gsr_forward_static" if raw_rest is None else "gsr_forward_static_raw", mask_render,
                              keep)
    args = (cap, _ptr(state.geom), gbytes, _ptr(state.binning), bbytes, _ptr(state.img), ibytes, _ptr(state.radii),
            _ptr(color), _ptr(depth), C.c_void_p(status.data_ptr())) + mr + (st,)
    if raw_rest is not None:
        rc = _lib.RawCloud(P, c.means3D, c.opacities, c.shs, _ptr(raw_rest), c.scales, c.rotations)
        _lib.check(fn(C.byref(s), C.byref(rc), *args), name)
    else:
        _lib.check(fn(C.byref(s), C.byref(c), *args), name)
    return color, depth


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings, return_alpha=False, camera_grad=False, depth_grad=False, deterministic=False,
                        static=None, mask_render=None):
    rs = raster_settings
    if mask_render is not None:   # uint8 [P]: the mask image as a trailing output; always the longest argument form
        cam = (rs.viewmatrix, rs.projmatrix, rs.campos) if camera_grad else (None, None, None)
        return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                         cov3Ds_precomp, rs, return_alpha, *cam, bool(depth_grad), bool(deterministic),
                                         static, mask_render)
    if static is not None:   # (capacity, status): gsr_forward_static; always the long argument form
        cam = (rs.viewmatrix, rs.projmatrix, rs.campos) if camera_grad else (None, None, None)
        return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                         cov3Ds_precomp, rs, return_alpha, *cam, bool(depth_grad), bool(deterministic),
                                         static)
    if depth_grad or deterministic:
        # depth_grad: the depth output's gradient is used (gsr_backward_depth); without it, it is dropped as in the
        # reference. deterministic: bit-reproducible backward (gsr_backward_deterministic).
        cam = (rs.viewmatrix, rs.projmatrix, rs.campos) if camera_grad else (None, None, None)
        return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                         cov3Ds_precomp, rs, return_alpha, *cam, bool(depth_grad), bool(deterministic))
    if camera_grad:   # the camera arrays become autograd inputs of the node (they are read from the settings as usual)
        return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                         cov3Ds_precomp, rs, return_alpha, rs.viewmatrix, rs.projmatrix, rs.campos)
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, return_alpha)


def _alpha_image(lib, state, device):
    """alpha = 1 - final_T as a [1,H,W] tensor (gsr_alpha_image; final_T is the reference's accum_alpha)."""
    alpha = torch.zeros(1, state.H, state.W, dtype=torch.float32, device=device)
    if state.P > 0 and state.W * state.H > 0:
        st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(lib.gsr_alpha_image(_ptr(state.img), state.img.numel(), state.W, state.H, _ptr(alpha), st),
                   "gsr_alpha_image")
    return alpha


def _mask_render_out(mask_render, rs, device):
    """(mask, out) for _forward_impl, with out the mask image [3,H,W] to be written; None without a mask."""
    if mask_render is None:
        return None
    return mask_render, torch.empty(3, int(rs.image_height), int(rs.image_width), dtype=torch.float32, device=device)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, return_alpha=False, viewmatrix=None, projmatrix=None, campos=None, depth_grad=False,
                deterministic=None, static=None, mask_render=None):
        mr = _mask_render_out(mask_render, raster_settings, means3D.device)
        color, depth, state, inputs = _forward_impl(means3D, sh, colors_precomp, opacities, scales, rotations,
                                                    cov3Ds_precomp, raster_settings, static=static, mask_render=mr)
        ctx.static_form = static is not None
        ctx.mask_form = mr is not None   # the mask image is a trailing output without a gradient
        ctx.return_alpha = bool(return_alpha)
        ctx.raster_settings = raster_settings
        ctx.camera_grad = viewmatrix is not None
        ctx.depth_grad = bool(depth_grad)
        ctx.long_form = deterministic is not None   # called with depth_grad and deterministic given
        ctx.deterministic = bool(deterministic)
        ctx.n_inputs = 10 + (3 if ctx.camera_grad else 0)
        if ctx.depth_grad:
            # outputs without a gradient arrive as None: no depth gradient -> the ordinary backward, and a loss on the
            # depth alone leaves the colour gradient None (treated as zeros)
            ctx.set_materialize_grads(False)
        ctx.state = state
        ctx.save_for_backward(*inputs, state.radii, state.geom, state.binning, state.img)
        ctx.mark_non_differentiable(state.radii)
        _RasterizeGaussians.last_state = state  # for parity tests / instrumentation only
        out = (color, state.radii, depth)
        if return_alpha:   # opt-in fourth output (not in the reference's tuple): alpha = 1 - final_T, differentiable
            with torch.cuda.device(means3D.device):
                out = out + (_alpha_image(_lib.load(), state, means3D.device),)
        if mr is not None:
            ctx.mark_non_differentiable(mr[1])
            out = out + (mr[1],)
        return out

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, *grad_rest):
        grad_alpha = grad_rest[0] if ctx.return_alpha else None   # the mask image's (last) entry is ignored
        lib = _lib.load()
        rs = ctx.raster_settings
        state = ctx.state
        (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, radii, geom, binning,
         img) = ctx.saved_tensors
        device = means3D.device
        P, M, W, H = state.P, state.M, state.W, state.H
        with torch.cuda.device(device):
            if grad_out_color is None:   # depth_grad: only the depth and/or alpha outputs carry a loss
                grad_out_color = torch.zeros(3, H, W, dtype=torch.float32, device=device)
            grad_out_color = _f32c(grad_out_color, device)
            f32 = dict(dtype=torch.float32, device=device)
            dL_dmeans3D = torch.empty(P, 3, **f32); dL_dmeans2D = torch.empty(P, 3, **f32)
            dL_dcolors = torch.empty(P, 3, **f32); dL_dopacity = torch.empty(P, 1, **f32)
            dL_dcov3D = torch.empty(P, 6, **f32); dL_dsh = torch.empty(P, M, 3, **f32)
            dL_dscales = torch.empty(P, 3, **f32); dL_drotations = torch.empty(P, 4, **f32)
            if P > 0:
                keep = []
                s = _make_settings(rs, M, device, keep)
                c = _make_cloud(P, means3D, opacities, sh, colors_precomp, scales, rotations, cov3Ds_precomp)
                sbytes = lib.gsr_backward_scratch_bytes(P)
                scratch = torch.empty(sbytes, dtype=torch.uint8, device=device)
                gr = _lib.Grads(_ptr(dL_dmeans3D), _ptr(dL_dmeans2D), _ptr(dL_dcolors), _ptr(dL_dopacity),
                                _ptr(dL_dcov3D), _ptr(dL_dsh), _ptr(dL_dscales), _ptr(dL_drotations))
                st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
                if ctx.deterministic:   # one entry point for every combination of alpha, camera and depth gradients
                    gd = _f32c(grad_depth, device) if ctx.depth_grad and grad_depth is not None else None
                    ga = None if grad_alpha is None else _f32c(grad_alpha, device)
                    cam = None
                    if ctx.camera_grad:
                        d_view = torch.empty(16, **f32); d_proj = torch.empty(16, **f32); d_cam = torch.empty(3, **f32)
                        cbytes = lib.gsr_camera_scratch_bytes(P)
                        cscratch = torch.empty(cbytes, dtype=torch.uint8, device=device)
                        cam = _lib.CameraGrads(_ptr(d_view), _ptr(d_proj), _ptr(d_cam), _ptr(cscratch), cbytes)
                        cam_grads = (d_view.view(rs.viewmatrix.shape), d_proj.view(rs.projmatrix.shape),
                                     d_cam.view(rs.campos.shape))
                    dbytes = lib.gsr_deterministic_scratch_bytes(P, state.cap, 0)
                    dscratch = torch.empty(dbytes, dtype=torch.uint8, device=device)
                    _lib.check(lib.gsr_backward_deterministic(C.byref(s), C.byref(c), state.cap, _ptr(geom), geom.numel(),
                                                              _ptr(binning), binning.numel(), _ptr(img), img.numel(),
                                                              _ptr(radii), _ptr(grad_out_color), _ptr(ga), _ptr(gd),
                                                              _ptr(scratch), sbytes, C.byref(gr),
                                                              None if cam is None else C.byref(cam), _ptr(dscratch),
                                                              dbytes, st), "gsr_backward_deterministic")
                elif ctx.depth_grad and grad_depth is not None:
                    gd = _f32c(grad_depth, device)
                    ga = None if grad_alpha is None else _f32c(grad_alpha, device)
                    cam = None
                    if ctx.camera_grad:
                        d_view = torch.empty(16, **f32); d_proj = torch.empty(16, **f32); d_cam = torch.empty(3, **f32)
                        cbytes = lib.gsr_camera_scratch_bytes(P)
                        cscratch = torch.empty(cbytes, dtype=torch.uint8, device=device)
                        cam = _lib.CameraGrads(_ptr(d_view), _ptr(d_proj), _ptr(d_cam), _ptr(cscratch), cbytes)
                        cam_grads = (d_view.view(rs.viewmatrix.shape), d_proj.view(rs.projmatrix.shape),
                                     d_cam.view(rs.campos.shape))
                    _lib.check(lib.gsr_backward_depth(C.byref(s), C.byref(c), state.cap, _ptr(geom), geom.numel(),
                                                      _ptr(binning), binning.numel(), _ptr(img), img.numel(),
                                                      _ptr(radii), _ptr(grad_out_color), _ptr(ga), _ptr(gd),
                                                      _ptr(scratch), sbytes, C.byref(gr),
                                                      None if cam is None else C.byref(cam), st), "gsr_backward_depth")
                elif ctx.camera_grad:
                    d_view = torch.empty(16, **f32); d_proj = torch.empty(16, **f32); d_cam = torch.empty(3, **f32)
                    cbytes = lib.gsr_camera_scratch_bytes(P)
                    cscratch = torch.empty(cbytes, dtype=torch.uint8, device=device)
                    cam = _lib.CameraGrads(_ptr(d_view), _ptr(d_proj), _ptr(d_cam), _ptr(cscratch), cbytes)
                    ga = None if grad_alpha is None else _f32c(grad_alpha, device)
                    _lib.check(lib.gsr_backward_camera(C.byref(s), C.byref(c), state.cap, _ptr(geom), geom.numel(),
                                                       _ptr(binning), binning.numel(), _ptr(img), img.numel(),
                                                       _ptr(radii), _ptr(grad_out_color), _ptr(ga), _ptr(scratch), sbytes,
                                                       C.byref(gr), C.byref(cam), st), "gsr_backward_camera")
                    cam_grads = (d_view.view(rs.viewmatrix.shape), d_proj.view(rs.projmatrix.shape),
                                 d_cam.view(rs.campos.shape))
                elif grad_alpha is not None:
                    grad_alpha = _f32c(grad_alpha, device)
                    _lib.check(lib.gsr_backward_alpha(C.byref(s), C.byref(c), state.cap, _ptr(geom), geom.numel(),
                                                      _ptr(binning), binning.numel(), _ptr(img), img.numel(),
                                                      _ptr(radii), _ptr(grad_out_color), _ptr(grad_alpha),
                                                      _ptr(scratch), sbytes, C.byref(gr), st), "gsr_backward_alpha")
                else:
                    _lib.check(lib.gsr_backward(C.byref(s), C.byref(c), state.cap, _ptr(geom), geom.numel(),
                                                _ptr(binning), binning.numel(), _ptr(img), img.numel(), _ptr(radii),
                                                _ptr(grad_out_color), _ptr(scratch), sbytes, C.byref(gr), st),
                               "gsr_backward")
                if scales.numel() == 0:  # cov3D_precomp path: the reference leaves these at their zero-fill
                    dL_dscales.zero_(); dL_drotations.zero_()
        # same slots as the reference (__init__.py:213-223); autograd drops grads of inputs that do not need one
        grads = (dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D,
                 None, None)
        if ctx.camera_grad:
            if P == 0:
                z = lambda t: torch.zeros_like(t, dtype=torch.float32)
                cam_grads = (z(rs.viewmatrix), z(rs.projmatrix), z(rs.campos))
            grads = grads + cam_grads
        if ctx.long_form:   # depth_grad, deterministic
            grads = grads + ((None, None, None) if not ctx.camera_grad else ()) + (None, None)
        if ctx.static_form or ctx.mask_form:
            grads = grads + (None,)
        if ctx.mask_form:
            grads = grads + (None,)
        return grads


class _RasterizeGaussiansRaw(torch.autograd.Function):
    """Fused-activation variant (SURVEY 8(f-3), gsr_forward_preprocess_raw / gsr_backward_raw): takes the scene model's
    raw parameters, gradients come back w.r.t. them."""

    @staticmethod
    def forward(ctx, means3D, means2D, opacity_logits, features_dc, features_rest, log_scales, raw_rotations,
                raster_settings, depth_grad=False, deterministic=None, static=None, mask_render=None):
        empty = torch.empty(0, dtype=torch.float32, device=means3D.device)
        mr = _mask_render_out(mask_render, raster_settings, means3D.device)
        color, depth, state, inputs = _forward_impl(means3D, features_dc, empty, opacity_logits, log_scales,
                                                    raw_rotations, empty, raster_settings, raw_rest=features_rest,
                                                    static=static, mask_render=mr)
        ctx.static_form = static is not None
        ctx.mask_form = mr is not None
        ctx.raster_settings = raster_settings
        ctx.state = state
        ctx.depth_grad = bool(depth_grad)
        ctx.long_form = deterministic is not None   # called with depth_grad and deterministic given
        ctx.deterministic = bool(deterministic)
        if ctx.depth_grad:   # as _RasterizeGaussians: None = no gradient for that output
            ctx.set_materialize_grads(False)
        (m3, dc, _, op, sc, ro, _, rest) = inputs
        ctx.save_for_backward(m3, dc, rest, op, sc, ro, state.radii, state.geom, state.binning, state.img)
        ctx.mark_non_differentiable(state.radii)
        _RasterizeGaussians.last_state = state
        if mr is not None:
            ctx.mark_non_differentiable(mr[1])
            return color, state.radii, depth, mr[1]
        return color, state.radii, depth

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_mask_render=None):
        lib = _lib.load()
        rs, state = ctx.raster_settings, ctx.state
        (means3D, dc, rest, logits, log_scales, raw_rot, radii, geom, binning, img) = ctx.saved_tensors
        device = means3D.device
        P, M = state.P, state.M
        with torch.cuda.device(device):
            if grad_out_color is None:   # depth_grad: a loss on the depth alone
                grad_out_color = torch.zeros(3, state.H, state.W, dtype=torch.float32, device=device)
            grad_out_color = _f32c(grad_out_color, device)
            f32 = dict(dtype=torch.float32, device=device)
            d_m3 = torch.empty(P, 3, **f32); d_m2 = torch.empty(P, 3, **f32); d_op = torch.empty(P, 1, **f32)
            d_dc = torch.empty(P, 1, 3, **f32); d_rest = torch.empty(P, M - 1, 3, **f32)
            d_sc = torch.empty(P, 3, **f32); d_ro = torch.empty(P, 4, **f32)
            if P > 0:
                keep = []
                s = _make_settings(rs, M, device, keep)
                rc = _lib.RawCloud(P, _ptr(means3D), _ptr(logits), _ptr(dc), _ptr(rest), _ptr(log_scales), _ptr(raw_rot))
                gr = _lib.RawGrads(_ptr(d_m3), _ptr(d_m2), _ptr(d_op), _ptr(d_dc), _ptr(d_rest), _ptr(d_sc), _ptr(d_ro))
                sbytes = lib.gsr_backward_scratch_bytes(P)
                scratch = torch.empty(sbytes, dtype=torch.uint8, device=device)
                st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
                if ctx.deterministic:
                    gd = _f32c(grad_depth, device) if ctx.depth_grad and grad_depth is not None else None
                    dbytes = lib.gsr_deterministic_scratch_bytes(P, state.cap, 0)
                    dscratch = torch.empty(dbytes, dtype=torch.uint8, device=device)
                    _lib.check(lib.gsr_backward_raw_deterministic(C.byref(s), C.byref(rc), state.cap, _ptr(geom),
                                                                  geom.numel(), _ptr(binning), binning.numel(), _ptr(img),
                                                                  img.numel(), _ptr(radii), _ptr(grad_out_color),
                                                                  _ptr(gd), _ptr(scratch), sbytes, C.byref(gr),
                                                                  _ptr(dscratch), dbytes, st),
                               "gsr_backward_raw_deterministic")
                elif ctx.depth_grad and grad_depth is not None:
                    gd = _f32c(grad_depth, device)
                    _lib.check(lib.gsr_backward_raw_depth(C.byref(s), C.byref(rc), state.cap, _ptr(geom), geom.numel(),
                                                          _ptr(binning), binning.numel(), _ptr(img), img.numel(),
                                                          _ptr(radii), _ptr(grad_out_color), _ptr(gd),
                                                          _ptr(scratch), sbytes, C.byref(gr), st), "gsr_backward_raw_depth")
                else:
                    _lib.check(lib.gsr_backward_raw(C.byref(s), C.byref(rc), state.cap, _ptr(geom), geom.numel(),
                                                    _ptr(binning), binning.numel(), _ptr(img), img.numel(), _ptr(radii),
                                                    _ptr(grad_out_color), _ptr(scratch), sbytes, C.byref(gr), st),
                               "gsr_backward_raw")
        if ctx.mask_form:   # depth_grad, deterministic, static, mask_render
            return d_m3, d_m2, d_op, d_dc, d_rest, d_sc, d_ro, None, None, None, None, None
        if ctx.static_form:   # depth_grad, deterministic, static
            return d_m3, d_m2, d_op, d_dc, d_rest, d_sc, d_ro, None, None, None, None
        if ctx.long_form:   # depth_grad, deterministic
            return d_m3, d_m2, d_op, d_dc, d_rest, d_sc, d_ro, None, None, None
        if ctx.depth_grad:
            return d_m3, d_m2, d_op, d_dc, d_rest, d_sc, d_ro, None, None
        return d_m3, d_m2, d_op, d_dc, d_rest, d_sc, d_ro, None


def _masked_scratch(lib, state, ctx, device):
    """(det_scratch, bytes, mask_scratch, bytes) of a masked backward; the first[] scratch stays on the forward state
    (``state.mask_first``, int32 [Ntile]) for tests and instrumentation."""
    u8 = dict(dtype=torch.uint8, device=device)
    dscratch, dbytes = None, 0
    if ctx.deterministic:
        dbytes = lib.gsr_deterministic_scratch_bytes(state.P, state.cap, 0)
        dscratch = torch.empty(dbytes, **u8)
    mbytes = lib.gsr_grad_mask_scratch_bytes(state.W, state.H)
    mscratch = torch.empty(mbytes, **u8)
    state.mask_first = mscratch
    return dscratch, dbytes, mscratch, mbytes


class _RasterizeGaussiansMasked(torch.autograd.Function):
    """``GaussianRasterizer(grad_mask=...)`` on ``forward``: the forward of _RasterizeGaussians, and one backward through
    gsr_backward_masked for every combination of alpha, depth, deterministic mode and static capacity. The mask is kept
    on the node as given (not saved for backward): the backward reads whatever it holds then."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, return_alpha, depth_grad, deterministic, static, grad_mask, mask_render=None):
        out = _RasterizeGaussians.forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                          cov3Ds_precomp, raster_settings, return_alpha, None, None, None, depth_grad,
                                          deterministic, static, mask_render)
        ctx.grad_mask = grad_mask
        return out

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, *grad_rest):
        grad_alpha = grad_rest[0] if ctx.return_alpha else None   # the mask image's (last) entry is ignored
        lib = _lib.load()
        rs, state = ctx.raster_settings, ctx.state
        (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, radii, geom, binning,
         img) = ctx.saved_tensors
        device = means3D.device
        P, M, W, H = state.P, state.M, state.W, state.H
        with torch.cuda.device(device):
            if grad_out_color is None:   # depth_grad: only the depth and/or alpha outputs carry a loss
                grad_out_color = torch.zeros(3, H, W, dtype=torch.float32, device=device)
            grad_out_color = _f32c(grad_out_color, device)
            f32 = dict(dtype=torch.float32, device=device)
            dL_dmeans3D = torch.empty(P, 3, **f32); dL_dmeans2D = torch.empty(P, 3, **f32)
            dL_dcolors = torch.empty(P, 3, **f32); dL_dopacity = torch.empty(P, 1, **f32)
            dL_dcov3D = torch.empty(P, 6, **f32); dL_dsh = torch.empty(P, M, 3, **f32)
            dL_dscales = torch.empty(P, 3, **f32); dL_drotations = torch.empty(P, 4, **f32)
            if P > 0:
                keep = []
                s = _make_settings(rs, M, device, keep)
                c = _make_cloud(P, means3D, opacities, sh, colors_precomp, scales, rotations, cov3Ds_precomp)
                sbytes = lib.gsr_backward_scratch_bytes(P)
                scratch = torch.empty(sbytes, dtype=torch.uint8, device=device)
                gr = _lib.Grads(_ptr(dL_dmeans3D), _ptr(dL_dmeans2D), _ptr(dL_dcolors), _ptr(dL_dopacity),
                                _ptr(dL_dcov3D), _ptr(dL_dsh), _ptr(dL_dscales), _ptr(dL_drotations))
                st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
                gd = _f32c(grad_depth, device) if ctx.depth_grad and grad_depth is not None else None
                ga = None if grad_alpha is None else _f32c(grad_alpha, device)
                dscratch, dbytes, mscratch, mbytes = _masked_scratch(lib, state, ctx, device)
                _lib.check(lib.gsr_backward_masked(C.byref(s), C.byref(c), state.cap, _ptr(geom), geom.numel(),
                                                   _ptr(binning), binning.numel(), _ptr(img), img.numel(), _ptr(radii),
                                                   _ptr(grad_out_color), _ptr(ga), _ptr(gd), _ptr(scratch), sbytes,
                                                   C.byref(gr), None, _ptr(dscratch), dbytes, _ptr(ctx.grad_mask),
                                                   _ptr(mscratch), mbytes, st), "gsr_backward_masked")
                if scales.numel() == 0:  # cov3D_precomp path: the reference leaves these at their zero-fill
                    dL_dscales.zero_(); dL_drotations.zero_()
        return (dL_dmeans3D, dL_dmeans2D, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D,
                None, None, None, None, None, None) + ((None,) if ctx.mask_form else ())


class _RasterizeGaussiansRawMasked(torch.autograd.Function):
    """``GaussianRasterizer(grad_mask=...)`` on ``forward_raw``: the forward of _RasterizeGaussiansRaw, the backward
    through gsr_backward_raw_masked."""

    @staticmethod
    def forward(ctx, means3D, means2D, opacity_logits, features_dc, features_rest, log_scales, raw_rotations,
                raster_settings, depth_grad, deterministic, static, grad_mask, mask_render=None):
        out = _RasterizeGaussiansRaw.forward(ctx, means3D, means2D, opacity_logits, features_dc, features_rest,
                                             log_scales, raw_rotations, raster_settings, depth_grad, deterministic,
                                             static, mask_render)
        ctx.grad_mask = grad_mask
        return out

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_mask_render=None):
        lib = _lib.load()
        rs, state = ctx.raster_settings, ctx.state
        (means3D, dc, rest, logits, log_scales, raw_rot, radii, geom, binning, img) = ctx.saved_tensors
        device = means3D.device
        P, M = state.P, state.M
        with torch.cuda.device(device):
            if grad_out_color is None:   # depth_grad: a loss on the depth alone
                grad_out_color = torch.zeros(3, state.H, state.W, dtype=torch.float32, device=device)
            grad_out_color = _f32c(grad_out_color, device)
            f32 = dict(dtype=torch.float32, device=device)
            d_m3 = torch.empty(P, 3, **f32); d_m2 = torch.empty(P, 3, **f32); d_op = torch.empty(P, 1, **f32)
            d_dc = torch.empty(P, 1, 3, **f32); d_rest = torch.empty(P, M - 1, 3, **f32)
            d_sc = torch.empty(P, 3, **f32); d_ro = torch.empty(P, 4, **f32)
            if P > 0:
                keep = []
                s = _make_settings(rs, M, device, keep)
                rc = _lib.RawCloud(P, _ptr(means3D), _ptr(logits), _ptr(dc), _ptr(rest), _ptr(log_scales), _ptr(raw_rot))
                gr = _lib.RawGrads(_ptr(d_m3), _ptr(d_m2), _ptr(d_op), _ptr(d_dc), _ptr(d_rest), _ptr(d_sc), _ptr(d_ro))
                sbytes = lib.gsr_backward_scratch_bytes(P)
                scratch = torch.empty(sbytes, dtype=torch.uint8, device=device)
                st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
                gd = _f32c(grad_depth, device) if ctx.depth_grad and grad_depth is not None else None
                dscratch, dbytes, mscratch, mbytes = _masked_scratch(lib, state, ctx, device)
                _lib.check(lib.gsr_backward_raw_masked(C.byref(s), C.byref(rc), state.cap, _ptr(geom), geom.numel(),
                                                       _ptr(binning), binning.numel(), _ptr(img), img.numel(),
                                                       _ptr(radii), _ptr(grad_out_color), _ptr(gd), _ptr(scratch),
                                                       sbytes, C.byref(gr), None, _ptr(dscratch), dbytes,
                                                       _ptr(ctx.grad_mask), _ptr(mscratch), mbytes, st),
                           "gsr_backward_raw_masked")
        return (d_m3, d_m2, d_op, d_dc, d_rest, d_sc, d_ro, None, None, None, None, None) + (
            (None,) if ctx.mask_form else ())


def _check_grad_mask(mask, camera_grad, raster_settings, name="grad_mask"):
    """Constructor checks of ``grad_mask`` (or, by ``name``, of another per-Gaussian mask such as ``mask_render``);
    returns the mask as uint8 (a bool mask is viewed, not copied)."""
    if not isinstance(mask, torch.Tensor):
        raise ValueError(f"{name} must be a torch.Tensor, got {type(mask).__name__}")
    if mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"{name} must be a bool or uint8 tensor, got {mask.dtype}")
    if mask.dim() != 1:
        raise ValueError(f"{name} must be 1-D [P], got shape {tuple(mask.shape)}")
    if not mask.is_cuda:
        raise ValueError(f"{name} must be on the rasterizer's CUDA device, got {mask.device}")
    view = getattr(raster_settings, "viewmatrix", None)
    if isinstance(view, torch.Tensor) and view.is_cuda and view.device != mask.device:
        raise ValueError(f"{name} is on {mask.device}, the camera on {view.device}")
    if not mask.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if camera_grad:
        raise ValueError(f"{name} cannot be combined with camera_grad: the camera gradient sums over every Gaussian")
    return mask.view(torch.uint8) if mask.dtype == torch.bool else mask


def mark_visible(rs, positions):
    """Frustum test of `positions` [P,3] under the camera of `rs` -> bool [P] (GaussianRasterizer.markVisible)."""
    # __init__.py:248-256 / rasterize_points.cu:159-175
    lib = _lib.load()
    with torch.no_grad():
        device = positions.device
        positions = _f32c(positions, device)
        P = positions.size(0)
        visible = torch.zeros(P, dtype=torch.bool, device=device)
        if P > 0:
            with torch.cuda.device(device):
                view = _f32c(rs.viewmatrix, device); proj = _f32c(rs.projmatrix, device)
                st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
                _lib.check(lib.gsr_mark_visible(P, _ptr(positions), _ptr(view), _ptr(proj), _ptr(visible), st),
                           "gsr_mark_visible")
    return visible


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings, return_alpha: bool = False, camera_grad: bool = False, depth_grad: bool = False,
                 deterministic=None, static_capacity=None, grad_mask=None, mask_render=None):
        """``return_alpha=True`` (opt-in, not in the reference) appends a fourth output to ``forward``: the alpha image
        ``1 - final_T`` [1,H,W] (the reference keeps final_T as ``accum_alpha`` but never returns it); it is
        differentiable like the colour.
        ``camera_grad=True`` (opt-in, not in the reference): ``raster_settings.viewmatrix / projmatrix / campos`` become
        differentiable inputs -- their ``.grad`` is filled by the backward (gsr_backward_camera), each array treated as an
        independent input exactly as the forward reads it.
        ``depth_grad=True`` (opt-in, for ``forward`` and ``forward_raw``): the depth output becomes differentiable
        (gsr_backward_depth). By default its gradient is dropped, as in the reference. When the depth receives no
        gradient the ordinary backward runs; a loss on the depth alone works too.
        ``deterministic`` (for ``forward``, ``forward_raw`` and ``apply_weights``): ``True`` computes the backward and
        ``apply_weights`` without float atomics (gsr_backward_deterministic), so two calls on the same inputs give the
        same bits; ``False`` keeps the faster default. ``None`` (default) follows
        ``torch.are_deterministic_algorithms_enabled()`` at the time of the call, so ``torch.use_deterministic_algorithms
        (True)`` (Lightning's ``trainer.deterministic=true``) selects it without other changes. Forward outputs are the
        same in both modes.
        ``static_capacity`` (opt-in, for ``forward`` and ``forward_raw``; an int > 0): the forward is sized for at most
        that many (Gaussian, tile) instances and never reads the count on the host: it only enqueues work, without a
        host synchronisation or a pinned allocation, so the call (and its backward) can be captured with
        ``torch.cuda.graph`` and the host can run ahead of the GPU. Each call writes ``self.status``, a device int32[2]
        tensor ``{num_rendered, num_rendered > static_capacity}``. When the capacity is too small the frame is EMPTY:
        colour = background, depth = 0, alpha = 0 and all gradients zero. Nothing checks this implicitly: call
        ``check_capacity()`` (it synchronises) where a synchronisation is acceptable. Outputs and radii are the same as
        without the option while the capacity suffices; ``apply_weights`` keeps its exact, host-sized path. Not
        combinable with ``raster_settings.debug`` (which synchronises after every launch).
        ``grad_mask`` (opt-in, for ``forward`` and ``forward_raw``; a bool or uint8 CUDA tensor [P]): only the Gaussians
        with ``grad_mask[i] != 0`` take gradients. Every gradient row of the others -- means3D, means2D, colours or SH,
        opacity, scales, rotations, cov3D, or the raw parameters -- is exactly +0.0, and the kernels skip their work
        (gsr_backward_masked): what GaussianEditor's ``apply_grad_mask`` hooks do after a full backward, but for all
        parameters, rotations included. The other rows equal the unmasked backward's: bit for bit when deterministic,
        to the rounding of the float atomics otherwise. The forward is unchanged. Combines with ``return_alpha``,
        ``depth_grad``, ``deterministic`` and ``static_capacity``; not with ``camera_grad`` (ValueError). The backward
        reads the tensor given here when it runs: changing it in place between forward and backward is the caller's
        business, as it is for the hooks.
        ``mask_render`` (opt-in, for ``forward`` and ``forward_raw``; a bool or uint8 CUDA tensor [P], usually the same
        tensor as ``grad_mask``): the forward appends one more output after everything it returns otherwise,
        ``(color, radii, depth[, alpha], mask_render)``, where ``mask_render`` [3,H,W] is the image of the Gaussians with
        ``mask_render[i] != 0`` drawn in white over the background -- the second forward GaussianEditor runs for its
        semantic map (``render(..., override_color=mask.float()[:, None].repeat(1, 3))["render"]``), bit for bit, but
        written by the same blend pass as the colour (gsr_forward_*_mask). Every other output and every gradient is
        unchanged; ``mask_render`` itself is not differentiable. Combines with every other option, ``camera_grad``
        included. On ``forward_raw`` the opacity is the in-kernel sigmoid of the logits, so the image matches that
        second forward on the activated parameters to the last bits only (the rounding note of INTEGRATION.md 5b)."""
        super().__init__()
        self.raster_settings = raster_settings
        self.return_alpha = bool(return_alpha)
        self.camera_grad = bool(camera_grad)
        self.depth_grad = bool(depth_grad)
        self.deterministic = None if deterministic is None else bool(deterministic)
        if static_capacity is not None:
            if isinstance(static_capacity, bool) or int(static_capacity) != static_capacity or not (
                    0 < int(static_capacity) < 2 ** 31):
                raise ValueError(f"static_capacity must be an int in [1, 2^31), got {static_capacity!r}")
            static_capacity = int(static_capacity)
        self.static_capacity = static_capacity
        self.status = None   # device int32[2] {num_rendered, overflow} of the last static-capacity call
        self.grad_mask = None if grad_mask is None else _check_grad_mask(grad_mask, self.camera_grad, raster_settings)
        self.mask_render = None if mask_render is None else _check_grad_mask(mask_render, False, raster_settings,
                                                                             "mask_render")

    def _grad_mask(self, means3D, name="grad_mask"):
        """The uint8 mask ``name`` (grad_mask or mask_render) for a forward on `means3D`, checked against its device and
        P; None when it is not set."""
        m = getattr(self, name)
        if m is None:
            return None
        if m.device != means3D.device:
            raise ValueError(f"{name} is on {m.device}, means3D on {means3D.device}")
        if m.numel() != means3D.size(0):
            raise ValueError(f"{name} has {m.numel()} entries for P = {means3D.size(0)} Gaussians")
        return m

    def _static(self, device):
        """(capacity, status) for a static-capacity call, or None. Raises before any launch on a debug setting."""
        if self.static_capacity is None:
            return None
        if self.raster_settings.debug:
            raise ValueError("static_capacity cannot be combined with debug=True: debug synchronises after every launch")
        if self.status is None or self.status.device != device:
            self.status = torch.zeros(2, dtype=torch.int32, device=device)
        return self.static_capacity, self.status

    def check_capacity(self):
        """Synchronise with the last static-capacity call and raise RuntimeError if its instance count exceeded
        ``static_capacity`` (that frame was rendered empty). Returns num_rendered otherwise."""
        if self.static_capacity is None or self.status is None:
            raise RuntimeError("check_capacity() needs a static_capacity rasterizer that has run a forward")
        R, over = (int(v) for v in self.status.cpu())
        if over:
            raise RuntimeError(f"num_rendered R={R} exceeds static_capacity={self.static_capacity}: the frame was "
                               f"rendered empty; raise the capacity to at least {R}")
        return R

    def _deterministic(self) -> bool:
        if self.deterministic is None:
            return torch.are_deterministic_algorithms_enabled()
        return self.deterministic

    def forward_raw(self, means3D, means2D, opacity_logits, features_dc, features_rest, log_scales, raw_rotations):
        """Opt-in fused-activation call (not part of the reference API): the arguments are the scene model's raw
        parameters (``_xyz, _opacity, _features_dc, _features_rest, _scaling, _rotation``); sigmoid / exp / normalize
        and the SH concatenation happen inside the preprocess kernels. Same return tuple as ``forward``."""
        det = self._deterministic()
        static = self._static(means3D.device)
        mr = self._grad_mask(means3D, "mask_render")
        if self.grad_mask is not None:
            return _RasterizeGaussiansRawMasked.apply(means3D, means2D, opacity_logits, features_dc, features_rest,
                                                      log_scales, raw_rotations, self.raster_settings, self.depth_grad,
                                                      det, static, self._grad_mask(means3D), *(() if mr is None else (mr,)))
        if mr is not None:
            return _RasterizeGaussiansRaw.apply(means3D, means2D, opacity_logits, features_dc, features_rest, log_scales,
                                                raw_rotations, self.raster_settings, self.depth_grad, det, static, mr)
        if static is not None:
            return _RasterizeGaussiansRaw.apply(means3D, means2D, opacity_logits, features_dc, features_rest, log_scales,
                                                raw_rotations, self.raster_settings, self.depth_grad, det, static)
        if self.depth_grad or det:
            return _RasterizeGaussiansRaw.apply(means3D, means2D, opacity_logits, features_dc, features_rest, log_scales,
                                                raw_rotations, self.raster_settings, self.depth_grad, det)
        return _RasterizeGaussiansRaw.apply(means3D, means2D, opacity_logits, features_dc, features_rest, log_scales,
                                            raw_rotations, self.raster_settings)

    def markVisible(self, positions):
        return mark_visible(self.raster_settings, positions)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        raster_settings = self.raster_settings

        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception("Please provide excatly one of either SHs or precomputed colors!")

        if ((scales is None or rotations is None) and cov3D_precomp is None) or (
            (scales is not None or rotations is not None) and cov3D_precomp is not None
        ):
            raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")

        static = self._static(means3D.device)
        empty = torch.empty(0, dtype=torch.float32, device=means3D.device)
        if shs is None:
            shs = empty
        if colors_precomp is None:
            colors_precomp = empty
        if scales is None:
            scales = empty
        if rotations is None:
            rotations = empty
        if cov3D_precomp is None:
            cov3D_precomp = empty

        mr = self._grad_mask(means3D, "mask_render")
        if self.grad_mask is not None:
            return _RasterizeGaussiansMasked.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                                   cov3D_precomp, raster_settings, self.return_alpha, self.depth_grad,
                                                   self._deterministic(), static, self._grad_mask(means3D),
                                                   *(() if mr is None else (mr,)))
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, raster_settings, self.return_alpha, self.camera_grad, self.depth_grad,
                                   self._deterministic(), static, mr)

    def apply_weights(self, means3D, means2D, opacities, shs=None, weights=None, scales=None, rotations=None,
                      cov3Ds_precomp=None, cnt=None, image_weights=None):
        """Semantic tracing (__init__.py:311-364): in-place accumulation into ``weights`` [P,CH] float32 and
        ``cnt`` [P,1] int32 from the 2-D mask ``image_weights`` [CH,H,W]."""
        assert weights is not None
        assert cnt is not None
        assert image_weights is not None
        lib = _lib.load()
        rs = self.raster_settings
        device = means3D.device
        empty = torch.empty(0, dtype=torch.float32, device=device)
        if not (weights.is_cuda and weights.dtype == torch.float32 and weights.is_contiguous()):
            raise RuntimeError("weights must be a contiguous float32 CUDA tensor (it is updated in place)")
        if not (cnt.is_cuda and cnt.dtype == torch.int32 and cnt.is_contiguous()):
            raise RuntimeError("cnt must be a contiguous int32 CUDA tensor (it is updated in place)")
        CH = int(image_weights.size(0))
        det = self._deterministic()
        with torch.no_grad():
            # the reference passes `weights` in the colors_precomp slot (rasterize_points.cu:223), so SH
            # evaluation is skipped; the forward's colours are never used
            # (any valid [P,3] float buffer will do for that slot -- means3D avoids an allocation)
            _, _, state, inputs = _forward_impl(means3D, empty, means3D, opacities, scales if scales is not None else empty,
                                                rotations if rotations is not None else empty,
                                                cov3Ds_precomp if cov3Ds_precomp is not None else empty, rs,
                                                render=False)
            if state.P == 0 or state.num_rendered == 0:
                return
            (m3, sh_, cp_, op_, sc_, ro_, cv_) = inputs
            with torch.cuda.device(device):
                keep = []
                s = _make_settings(rs, 0, device, keep)
                c = _make_cloud(state.P, m3, op_, sh_, cp_, sc_, ro_, cv_)
                iw = _f32c(image_weights, device)
                st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
                if det:   # bit-identical weights on every call (gsr_apply_weights_deterministic)
                    dbytes = lib.gsr_deterministic_scratch_bytes(state.P, state.num_rendered, CH)
                    dscratch = torch.empty(dbytes, dtype=torch.uint8, device=device)
                    _lib.check(lib.gsr_apply_weights_deterministic(
                        C.byref(s), C.byref(c), state.num_rendered, _ptr(state.geom), state.geom.numel(),
                        _ptr(state.binning), state.binning.numel(), _ptr(state.img), state.img.numel(), _ptr(state.radii),
                        _ptr(iw), CH, _ptr(weights), _ptr(cnt), _ptr(dscratch), dbytes, st),
                        "gsr_apply_weights_deterministic")
                    return
                _lib.check(lib.gsr_apply_weights(C.byref(s), C.byref(c), state.num_rendered, _ptr(state.geom),
                                                 state.geom.numel(), _ptr(state.binning), state.binning.numel(),
                                                 _ptr(state.img), state.img.numel(), _ptr(state.radii), _ptr(iw), CH,
                                                 _ptr(weights), _ptr(cnt), st), "gsr_apply_weights")


# ---- instrumentation for parity tests (not part of the reference API) ---------------------------------------
def forward_state_views(state: _ForwardState):
    """Decode the opaque workspaces of a forward into torch tensors (views onto the workspace memory)."""
    lib = _lib.load()
    P, R, W, H = state.P, state.num_rendered, state.W, state.H
    cap = state.cap
    out = {}

    def view(ptr, base: torch.Tensor, numel, dtype):
        off = ptr - base.data_ptr()
        nbytes = numel * torch.empty(0, dtype=dtype).element_size()
        return base[off:off + nbytes].view(dtype)

    if P == 0:
        dev = state.radii.device
        e = lambda dt, *shape: torch.empty(*shape, dtype=dt, device=dev)
        out.update(records=e(torch.float32, 0, 12), tiles_touched=e(torch.int32, 0), clamped=e(torch.uint8, 0),
                   depth_order=e(torch.int32, 0), point_list=e(torch.int32, 0), tile_keys=e(torch.int32, 0),
                   final_T=e(torch.float32, H, W), n_contrib=e(torch.int32, H, W),
                   ranges=torch.zeros(((W + 15) // 16) * ((H + 15) // 16), 2, dtype=torch.int32, device=dev))
        return out
    gv = _lib.GeometryView()
    _lib.check(lib.gsr_view_geometry(_ptr(state.geom), P, C.byref(gv)), "gsr_view_geometry")
    out["records"] = view(gv.records, state.geom, P * 12, torch.float32).view(P, 12)
    out["tiles_touched"] = view(gv.tiles_touched, state.geom, P, torch.int32)
    out["clamped"] = view(gv.clamped, state.geom, P, torch.uint8)
    out["depth_order"] = view(gv.depth_order, state.geom, P, torch.int32)
    iv = _lib.ImageView()
    _lib.check(lib.gsr_view_image(_ptr(state.img), W, H, C.byref(iv)), "gsr_view_image")
    ntile = ((W + 15) // 16) * ((H + 15) // 16)
    out["final_T"] = view(iv.final_T, state.img, W * H, torch.float32).view(H, W)
    out["n_contrib"] = view(iv.n_contrib, state.img, W * H, torch.int32).view(H, W)
    out["ranges"] = view(iv.ranges, state.img, ntile * 2, torch.int32).view(ntile, 2)
    if R > 0:
        bv = _lib.BinningView()
        _lib.check(lib.gsr_view_binning(_ptr(state.binning), P, cap, W, H, C.byref(bv)), "gsr_view_binning")
        out["point_list"] = view(bv.point_list, state.binning, R, torch.int32)
        out["tile_keys"] = view(bv.tile_keys, state.binning, R, torch.int16 if bv.tile_key_bytes == 2 else torch.int32)
    else:
        out["point_list"] = torch.empty(0, dtype=torch.int32, device=state.geom.device)
        out["tile_keys"] = torch.empty(0, dtype=torch.int32, device=state.geom.device)
    return out
