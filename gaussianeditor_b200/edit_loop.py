"""Config-5 harness: the SHAPE of one GaussianEditor edit-n2n training step around the rasterizer, with everything
that is not this repository's hot path stubbed (BASELINE.json configs[4], SURVEY.md 3.3 / 8(d)).

Per step, as threestudio/systems/GassuianEditor.py:155-224 + GassuianEditorEdit.py:64-150 + :251-281 do it:
  render(cam, gaussians, pipe, bg)                       forward #1 (SH colours, grad)
  render(cam, ..., override_color=mask)                  forward #2 (colors_precomp path; never back-propagated)
  loss = L1(render, cached edited frame of that view)    (InstructPix2Pix + LPIPS replaced by a fixed target)
  loss.backward()                                        one rasterizer backward
  densification stats from viewspace_points.grad, max_radii2D from radii
  every `densification_interval` steps: clone the top `max_densify_percent` by gradient, prune low opacity (P changes)
  Adam step over the six parameter groups (scene/gaussian_model.py:341-374)

`EditScene` is a minimal stand-in for the reference's GaussianModel (which cannot be imported on the GPU box: plyfile,
simple_knn and the reference tree are absent): same property names (`get_xyz`, `get_opacity`, `get_scaling`,
`get_rotation`, `get_features`, `active_sh_degree`, `max_sh_degree`, `mask`), same activations
(sigmoid / exp / normalize, scene/gaussian_model.py:47-58,221-258), so `gaussian_renderer.render()` consumes it exactly
as it consumes the real model.  The rasterizer implementation is injected, so the same loop runs on this repository's
kernels and on the reference's CUDA build (oracle/ref_torch.py) for the A/B render-time fraction.
"""
from __future__ import annotations

import math
import time
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn.functional as F

from . import synth
from .rasterizer import GaussianRasterizationSettings


class EditScene:
    def __init__(self, cloud: synth.Cloud, device):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
        eps = 1e-6
        self._xyz = t(cloud.means3D).requires_grad_(True)
        self._features_dc = t(cloud.shs[:, :1, :]).contiguous().requires_grad_(True)
        self._features_rest = t(cloud.shs[:, 1:, :]).contiguous().requires_grad_(True)
        self._scaling = torch.log(t(cloud.scales)).requires_grad_(True)
        self._rotation = t(cloud.rotations).requires_grad_(True)
        op = t(cloud.opacities).clamp(eps, 1 - eps)
        self._opacity = torch.log(op / (1 - op)).requires_grad_(True)
        self.active_sh_degree = self.max_sh_degree = cloud.sh_degree
        P = self._xyz.shape[0]
        d = self._xyz.detach().norm(dim=1)
        self.mask = d <= torch.quantile(d[: min(P, 1_000_000)], 0.2)   # "20 % of Gaussians nearest the origin"
        self.max_radii2D = torch.zeros(P, device=device)
        self.xyz_gradient_accum = torch.zeros(P, 1, device=device)
        self.denom = torch.zeros(P, 1, device=device)
        self._make_optimizer()

    def _params(self):
        return [("xyz", self._xyz, 1.6e-5), ("f_dc", self._features_dc, 2.5e-3), ("f_rest", self._features_rest, 1.25e-4),
                ("opacity", self._opacity, 0.1), ("scaling", self._scaling, 1e-2), ("rotation", self._rotation, 2e-3)]

    def _make_optimizer(self):
        self.optimizer = torch.optim.Adam([{"params": [p], "lr": lr, "name": n} for n, p, lr in self._params()], eps=1e-15)

    # -- the reference model's read API ---------------------------------------------------------------------
    @property
    def get_xyz(self): return self._xyz
    @property
    def get_opacity(self): return torch.sigmoid(self._opacity)
    @property
    def get_scaling(self): return torch.exp(self._scaling)
    @property
    def get_rotation(self): return F.normalize(self._rotation)
    @property
    def get_features(self): return torch.cat((self._features_dc, self._features_rest), dim=1)

    def add_densification_stats(self, viewspace_grad, update_filter):   # scene/gaussian_model.py:811-815
        self.xyz_gradient_accum[update_filter] += torch.norm(viewspace_grad[update_filter, :2], dim=-1, keepdim=True)
        self.denom[update_filter] += 1

    def densify_and_prune(self, max_densify_percent=0.01, min_opacity=0.005):
        """Clone the `max_densify_percent` Gaussians with the largest mean view-space gradient, prune those below
        `min_opacity` (shape of scene/gaussian_model.py:768-809; the split branch is folded into clone)."""
        with torch.no_grad():
            grads = (self.xyz_gradient_accum / self.denom.clamp_min(1)).squeeze(1)
            P = grads.numel()
            k = max(1, int(P * max_densify_percent))
            sel = torch.topk(grads, k).indices
            keep = (torch.sigmoid(self._opacity).squeeze(1) >= min_opacity)
            keep[sel] = True
            idx = torch.cat([torch.nonzero(keep).squeeze(1), sel])
            for name in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"):
                setattr(self, name, getattr(self, name).detach()[idx].clone().requires_grad_(True))
            self.mask = self.mask[idx]
            n = idx.numel()
            dev = self._xyz.device
            self.max_radii2D = torch.zeros(n, device=dev)
            self.xyz_gradient_accum = torch.zeros(n, 1, device=dev)
            self.denom = torch.zeros(n, 1, device=dev)
            self._make_optimizer()   # the reference re-stitches Adam state; the harness restarts it


def make_view(cam: synth.Camera, device):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy),
                           image_height=cam.image_height, image_width=cam.image_width,
                           world_view_transform=t(cam.viewmatrix), full_proj_transform=t(cam.projmatrix),
                           camera_center=t(cam.campos))


def run_edit_loop(rasterizer_cls, steps=200, P=None, device="cuda", densification_interval=100, seed=0,
                  log=None, fused_activations=False):
    """Returns a dict with total / render wall times (CUDA-event timed) and the per-step Gaussian counts.
    ``fused_activations`` renders the SH pass through ``render(..., fused_activations=True)`` (this repository's rasterizer only)."""
    from . import gaussian_renderer as GR
    cloud, cams = synth.make_config("c5", P=P)
    scene = EditScene(cloud, device)
    views = [make_view(c, device) for c in cams]
    pipe = SimpleNamespace(convert_SHs_python=False, compute_cov3D_python=False, debug=False)
    bg = torch.zeros(3, device=device)
    # the rasterizer class is injected by swapping the name render() resolves
    old = GR.GaussianRasterizer
    GR.GaussianRasterizer = rasterizer_cls
    ev = lambda: torch.cuda.Event(enable_timing=True)
    try:
        with torch.no_grad():   # "render_all_view": cached originals -> edited targets (guidance stub: + seeded noise)
            g = torch.Generator(device=device).manual_seed(seed)
            targets = []
            for v in views:
                img = GR.render(v, scene, pipe, bg)["render"]
                targets.append((img + 0.05 * torch.randn(img.shape, generator=g, device=device)).clamp(0, 1))
        render_ms = 0.0
        counts, losses, radii_trace = [], [], []
        rng = np.random.default_rng(seed)
        torch.cuda.synchronize()
        t_all0, t_all1 = ev(), ev()
        t_all0.record()
        pend = []
        for step in range(1, steps + 1):
            k = int(rng.integers(len(views)))
            e0, e1, e2, e3 = ev(), ev(), ev(), ev()
            e0.record()
            pkg = GR.render(views[k], scene, pipe, bg, fused_activations=fused_activations)       # forward #1
            sem = GR.render(views[k], scene, pipe, bg,
                            override_color=scene.mask[..., None].float().repeat(1, 3))["render"]  # forward #2
            e1.record()
            semantic = torch.norm(sem, dim=0) > 0.8                                               # thresholded: no grad
            loss = 10.0 * (pkg["render"] - targets[k]).abs().mean() + 0.0 * semantic.float().mean()
            scene.optimizer.zero_grad(set_to_none=True)
            e2.record()
            loss.backward()                                                                       # rasterizer backward
            e3.record()
            pend.append((e0, e1, e2, e3))
            with torch.no_grad():
                vis = pkg["visibility_filter"]
                scene.max_radii2D[vis] = torch.max(scene.max_radii2D[vis], pkg["radii"][vis].float())
                scene.add_densification_stats(pkg["viewspace_points"].grad, vis)
            scene.optimizer.step()
            losses.append(loss.detach())
            if step % densification_interval == 0 and step < steps:
                radii_trace.append(scene.max_radii2D.clone())   # what the reference's prune test reads (:790-795)
                scene.densify_and_prune()
            counts.append(scene._xyz.shape[0])
        t_all1.record()
        torch.cuda.synchronize()
        for e0, e1, e2, e3 in pend:   # backward time includes the few autograd elementwise kernels around it
            render_ms += e0.elapsed_time(e1) + e2.elapsed_time(e3)
        total_ms = t_all0.elapsed_time(t_all1)
    finally:
        GR.GaussianRasterizer = old
    return dict(steps=steps, total_ms=total_ms, render_ms=render_ms, render_fraction=render_ms / total_ms,
                ms_per_step=total_ms / steps, P_first=counts[0], P_last=counts[-1], final_loss=float(loss.detach()),
                counts=counts, losses=torch.stack(losses).cpu().tolist(), max_radii2D=scene.max_radii2D.cpu(),
                max_radii2D_at_densify=[r.cpu() for r in radii_trace])
