"""Host-side mirror of the reference's render boundary
(/root/reference/gaussiansplatting/gaussian_renderer/__init__.py: ``camera2rasterizer`` :21-42, ``render`` :45-150).

Same names, arguments, result dictionary and conventions, so GaussianEditor's edit/add/delete loops that call
``render(cam, gaussians, pipe, bg)`` work on top of this rasterizer without touching the callers.  The
optional Python-side SH->RGB / covariance paths of the reference (``pipe.convert_SHs_python`` /
``pipe.compute_cov3D_python``, both False in every GaussianEditor config, arguments/__init__.py:63-67) are
supported through the same rasterizer arguments.
"""
from __future__ import annotations

import math

import torch

from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer


def _settings_for(cam, bg_color, scale_modifier, sh_degree) -> GaussianRasterizationSettings:
    """The camera -> settings mapping both entry points share (FoV -> tangent, transposed matrices as stored by
    scene/cameras.py:92-94)."""
    fields = dict(image_height=int(cam.image_height), image_width=int(cam.image_width),
                  tanfovx=math.tan(0.5 * cam.FoVx), tanfovy=math.tan(0.5 * cam.FoVy), bg=bg_color,
                  scale_modifier=scale_modifier, viewmatrix=cam.world_view_transform,
                  projmatrix=cam.full_proj_transform, sh_degree=sh_degree, campos=cam.camera_center,
                  prefiltered=False, debug=False)
    return GaussianRasterizationSettings(**fields)


def camera2rasterizer(viewpoint_camera, bg_color: torch.Tensor, sh_degree: int = 0):
    return GaussianRasterizer(raster_settings=_settings_for(viewpoint_camera, bg_color, 1.0, sh_degree))


def _sh_basis(deg: int, d: torch.Tensor) -> torch.Tensor:
    """Real SH basis up to degree 3 at unit directions d [P,3] -> [P,(deg+1)^2], the reference's constants and signs
    (utils/sh_utils.py / cuda_rasterizer/forward.cu:20-71)."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    cols = [torch.full_like(x, 0.28209479177387814)]
    if deg >= 1:
        c1 = 0.4886025119029199
        cols += [-c1 * y, c1 * z, -c1 * x]
    if deg >= 2:
        xx, yy, zz = x * x, y * y, z * z
        cols += [1.0925484305920792 * x * y, -1.0925484305920792 * y * z, 0.31539156525252005 * (2 * zz - xx - yy),
                 -1.0925484305920792 * x * z, 0.5462742152960396 * (xx - yy)]
    if deg >= 3:
        cols += [-0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * x * y * z,
                 -0.4570457994644658 * y * (4 * zz - xx - yy), 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy),
                 -0.4570457994644658 * x * (4 * zz - xx - yy), 1.445305721320277 * z * (xx - yy),
                 -0.5900435899266435 * x * (xx - 3 * yy)]
    return torch.stack(cols, dim=1)


def _python_sh_colors(pc, camera_center) -> torch.Tensor:
    """``pipe.convert_SHs_python``: evaluate the SH colour in PyTorch and hand it over as precomputed colour
    (gaussian_renderer/__init__.py:103-121): clamp_min(sum_k basis_k * sh_k + 0.5, 0)."""
    feats = pc.get_features                                   # [P, M, 3]
    view = pc.get_xyz - camera_center.reshape(1, 3)
    view = view / view.norm(dim=1, keepdim=True)
    basis = _sh_basis(pc.active_sh_degree, view)              # [P, nb]
    rgb = torch.einsum("pk,pkc->pc", basis, feats[:, :basis.shape[1], :])
    return torch.clamp_min(rgb + 0.5, 0.0)


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None,
           fused_activations: bool = False):
    """Render the scene; background tensor must be on the GPU. Returns the reference's dictionary:
    render [3,H,W], viewspace_points [P,3] (grad sink for densification), visibility_filter, radii, depth_3dgs.

    ``fused_activations=True`` (opt-in, not in the reference; SURVEY 8(f-3)) hands the scene model's RAW parameters
    (``pc._opacity, pc._features_dc, pc._features_rest, pc._scaling, pc._rotation``) to the rasterizer, which applies
    sigmoid / exp / normalize and reads the SH row from the two feature arrays inside its preprocess kernels: the
    per-render PyTorch prologue (five elementwise kernels, a [P,16,3] ``torch.cat``) and its autograd epilogue go away.
    Only valid for the plain SH path (no override colour, no Python-side SH / covariance)."""
    xyz = pc.get_xyz
    # gradient sink for the 2-D means: densification reads its .grad (gaussian_renderer/__init__.py:60-69)
    screenspace_points = torch.zeros_like(xyz, requires_grad=True) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    rasterizer = GaussianRasterizer(
        raster_settings=_settings_for(viewpoint_camera, bg_color, scaling_modifier, pc.active_sh_degree))
    python_sh = getattr(pipe, "convert_SHs_python", False)
    python_cov = getattr(pipe, "compute_cov3D_python", False)

    if fused_activations:
        if override_color is not None or python_sh or python_cov:
            raise ValueError("fused_activations needs the plain SH + scale/rotation path")
        image, radii, depth = rasterizer.forward_raw(
            means3D=xyz, means2D=screenspace_points, opacity_logits=pc._opacity, features_dc=pc._features_dc,
            features_rest=pc._features_rest, log_scales=pc._scaling, raw_rotations=pc._rotation)
    else:
        kw = dict(means3D=xyz.float(), means2D=screenspace_points.float(), opacities=pc.get_opacity.float())
        if python_cov:
            kw["cov3D_precomp"] = pc.get_covariance(scaling_modifier)
        else:
            kw.update(scales=pc.get_scaling.float(), rotations=pc.get_rotation.float())
        if override_color is not None:
            kw["colors_precomp"] = override_color
        elif python_sh:
            kw["colors_precomp"] = _python_sh_colors(pc, viewpoint_camera.camera_center)
        else:
            kw["shs"] = pc.get_features.float()
        image, radii, depth = rasterizer(**kw)
    return {"render": image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0, "radii": radii,
            "depth_3dgs": depth}
