"""ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Python front-end of ``oracle/_ref/libdgr_ref.so``: the reference's OWN CUDA rasterizer sources
(/root/reference/gaussiansplatting/submodules/diff-gaussian-rasterization/cuda_rasterizer/*.cu), compiled
unmodified for sm_90a by ``oracle/Makefile`` (target ``ref``) behind the thin C shim ``oracle/ref_shim.cu``.
It restates only the reference's torch glue (rasterize_points.cu:35-157: output allocation, zero-filled
gradient tensors) so the reference kernels and host orchestration can run on the GPU box without building the
reference's torch extension.  Used by the GPU parity tests as THE primary oracle and by ``bench.py --impl
reference`` as the A/B baseline.  Needs a GPU; never imported by the product package.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libdgr_ref.so")
_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError(f"{LIB_PATH} missing: build() compiles it when the GaussianEditor checkout is present "
                               "($GSR_REFERENCE; or `make -C oracle ref REF=<checkout>/gaussiansplatting/submodules/"
                               "diff-gaussian-rasterization`)")
        L = C.CDLL(LIB_PATH)
        L.dgr_create.restype = C.c_void_p
        L.dgr_destroy.argtypes = [C.c_void_p]
        L.dgr_forward.restype = C.c_int
        L.dgr_forward.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int] + \
            [C.c_void_p] * 5 + [C.c_float] + [C.c_void_p] * 5 + [C.c_float, C.c_float, C.c_int] + [C.c_void_p] * 3
        L.dgr_backward.restype = None
        L.dgr_backward.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int] + \
            [C.c_void_p] * 4 + [C.c_float] + [C.c_void_p] * 5 + [C.c_float, C.c_float] + [C.c_void_p] * 11
        L.dgr_mark_visible.argtypes = [C.c_int] + [C.c_void_p] * 4
        L.dgr_apply_weights.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int] + \
            [C.c_void_p] * 5 + [C.c_float] + [C.c_void_p] * 5 + [C.c_float, C.c_float, C.c_int] + \
            [C.c_void_p] * 3 + [C.c_int]
        L.dgr_state_ptrs.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.dgr_last_cuda_error.restype = C.c_int
        L.dgr_copy_d2d.restype = C.c_int
        L.dgr_copy_d2d.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        _lib = L
    return _lib


def _p(t):
    return None if t is None or t.numel() == 0 else C.c_void_p(t.data_ptr())


class ReferenceRasterizer:
    """Runs on the legacy default stream like the reference; callers must be on torch's default stream."""

    def __init__(self):
        self.L = lib()
        self.ctx = C.c_void_p(self.L.dgr_create())

    def __del__(self):
        try:
            self.L.dgr_destroy(self.ctx)
        except Exception:
            pass

    def forward(self, *, means3D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, bg, viewmatrix,
                projmatrix, campos, tanfovx, tanfovy, image_height, image_width, sh_degree, scale_modifier=1.0):
        dev = means3D.device
        P = means3D.shape[0]
        M = shs.shape[1] if shs is not None and shs.numel() else 0
        H, W = int(image_height), int(image_width)
        # rasterize_points.cu:57-60
        out_color = torch.full((3, H, W), 0.0, dtype=torch.float32, device=dev)
        out_depth = torch.full((1, H, W), 0.0, dtype=torch.float32, device=dev)
        radii = torch.full((P,), 0, dtype=torch.int32, device=dev)
        R = 0
        if P:
            R = self.L.dgr_forward(self.ctx, P, int(sh_degree), M, _p(bg), W, H, _p(means3D), _p(shs),
                                   _p(colors_precomp), _p(opacities), _p(scales), float(scale_modifier), _p(rotations),
                                   _p(cov3D_precomp), _p(viewmatrix), _p(projmatrix), _p(campos), float(tanfovx),
                                   float(tanfovy), 0, _p(out_color), _p(out_depth), _p(radii))
        self.last = dict(P=P, M=M, H=H, W=W, R=R, D=int(sh_degree))
        return out_color, radii, out_depth, R

    def backward(self, *, dL_dcolor, radii, R, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, bg,
                 viewmatrix, projmatrix, campos, tanfovx, tanfovy, sh_degree, scale_modifier=1.0):
        dev = means3D.device
        P = means3D.shape[0]
        M = shs.shape[1] if shs is not None and shs.numel() else 0
        H, W = dL_dcolor.shape[1], dL_dcolor.shape[2]
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)  # rasterize_points.cu:120-128
        g = dict(dL_dmeans3D=z(P, 3), dL_dmeans2D=z(P, 3), dL_dcolors=z(P, 3), dL_dconic=z(P, 2, 2),
                 dL_dopacity=z(P, 1), dL_dcov3D=z(P, 6), dL_dsh=z(P, M, 3), dL_dscales=z(P, 3), dL_drotations=z(P, 4))
        if P:
            self.L.dgr_backward(self.ctx, P, int(sh_degree), M, int(R), _p(bg), W, H, _p(means3D), _p(shs),
                                _p(colors_precomp), _p(scales), float(scale_modifier), _p(rotations),
                                _p(cov3D_precomp), _p(viewmatrix), _p(projmatrix), _p(campos), float(tanfovx),
                                float(tanfovy), _p(radii), _p(dL_dcolor.contiguous()), _p(g["dL_dmeans2D"]),
                                _p(g["dL_dconic"]), _p(g["dL_dopacity"]), _p(g["dL_dcolors"]), _p(g["dL_dmeans3D"]),
                                _p(g["dL_dcov3D"]), _p(g["dL_dsh"]) if M else None, _p(g["dL_dscales"]),
                                _p(g["dL_drotations"]))
        return g

    def state(self):
        """Device views of the reference's intermediate buffers (decoded with its own fromChunk)."""
        d = self.last
        P, W, H, R = d["P"], d["W"], d["H"], d["R"]
        ptrs = (C.c_void_p * 13)()
        self.L.dgr_state_ptrs(self.ctx, P, W, H, R, ptrs)
        dev = torch.device("cuda", torch.cuda.current_device())

        def copy(ptr, numel, dtype):
            out = torch.empty(numel, dtype=dtype, device=dev)
            if numel and ptr:
                rc = self.L.dgr_copy_d2d(C.c_void_p(out.data_ptr()), C.c_void_p(ptr),
                                         C.c_size_t(out.numel() * out.element_size()))
                assert int(rc) == 0, rc
            return out
        ntile = ((W + 15) // 16) * ((H + 15) // 16)
        return dict(
            depths=copy(ptrs[0], P, torch.float32), clamped=copy(ptrs[1], 3 * P, torch.uint8).view(P, 3),
            means2D=copy(ptrs[2], 2 * P, torch.float32).view(P, 2), cov3D=copy(ptrs[3], 6 * P, torch.float32).view(P, 6),
            conic_opacity=copy(ptrs[4], 4 * P, torch.float32).view(P, 4), rgb=copy(ptrs[5], 3 * P, torch.float32).view(P, 3),
            point_offsets=copy(ptrs[6], P, torch.int32), tiles_touched=copy(ptrs[7], P, torch.int32),
            keys=copy(ptrs[8], R, torch.int64), point_list=copy(ptrs[9], R, torch.int32),
            ranges=copy(ptrs[10], 2 * ntile, torch.int32).view(ntile, 2),
            n_contrib=copy(ptrs[11], W * H, torch.int32).view(H, W),
            final_T=copy(ptrs[12], W * H, torch.float32).view(H, W))

    def mark_visible(self, means3D, viewmatrix, projmatrix):
        P = means3D.shape[0]
        present = torch.zeros(P, dtype=torch.bool, device=means3D.device)
        if P:
            self.L.dgr_mark_visible(P, _p(means3D), _p(viewmatrix), _p(projmatrix), _p(present))
        return present

    def apply_weights(self, *, means3D, opacities, scales, rotations, weights, cnt, image_weights, bg, viewmatrix,
                      projmatrix, campos, tanfovx, tanfovy, image_height, image_width, scale_modifier=1.0):
        P = means3D.shape[0]
        radii = torch.zeros(P, dtype=torch.int32, device=means3D.device)
        CH = image_weights.shape[0]
        if P:
            self.L.dgr_apply_weights(self.ctx, P, 0, 0, _p(bg), int(image_width), int(image_height), _p(means3D), None,
                                     _p(weights), _p(opacities), _p(scales), float(scale_modifier), _p(rotations), None,
                                     _p(viewmatrix), _p(projmatrix), _p(campos), float(tanfovx), float(tanfovy), 0,
                                     _p(image_weights.contiguous()), _p(radii), _p(cnt), CH)
