"""Config-5 harness: the SHAPE of one GaussianEditor edit-n2n training step around the rasterizer, with everything
that is not this repository's hot path stubbed (BASELINE.json configs[4], SURVEY.md 3.3 / 8(d)).

Per step, as threestudio/systems/GassuianEditor.py:155-224 + GassuianEditorEdit.py:64-150 + :251-281 do it:
  render(cam, gaussians, pipe, bg)                       forward #1 (SH colours, grad)
  render(cam, ..., override_color=mask)                  forward #2 (colors_precomp path; never back-propagated)
                                                         (semantic="fused": forward #1's mask_render output instead)
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

`run_edit_loop(..., cuda_graph=True)` captures the whole step (both forwards, loss, backward, densification stats and
``Adam(capturable=True)``) once per Gaussian count with ``torch.cuda.graph`` and replays it, on the rasterizer's
static-capacity forward; ``static_capacity=True`` runs the same step eagerly. Both never synchronise between
densification points.
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

# GaussianEditor's anchor-loss settings, as the bear edit script (SURVEY.md's edit shape) sets them
ANCHOR_WEIGHT_INIT_G0 = 0.01    # first weight of generation 0
ANCHOR_WEIGHT_INIT = 0.01       # first weight of every later generation
ANCHOR_WEIGHT_MULTIPLIER = 1.3  # every weight grows by this at each densification ...
MAX_ANCHOR_WEIGHT = 10          # ... up to this
ANCHOR_LAMBDA = {"loss_anchor_color": 0.0, "loss_anchor_geo": 50.0, "loss_anchor_opacity": 50.0,
                 "loss_anchor_scale": 50.0}
_ANCHOR_GROUP = {"_xyz": "loss_anchor_geo", "_rotation": "loss_anchor_geo", "_features_dc": "loss_anchor_color",
                 "_features_rest": "loss_anchor_color", "_opacity": "loss_anchor_opacity", "_scaling": "loss_anchor_scale"}


class EditScene:
    def __init__(self, cloud: synth.Cloud, device, capturable: bool = False, optimizer: str = "adam",
                 track_anchor: bool = False):
        self.capturable = capturable   # Adam(capturable=True): the optimizer step can be captured in a CUDA graph
        self.optimizer_kind = optimizer   # "adam": torch.optim.Adam, "masked": MaskedAdam on `mask`
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
        self.hooks = None   # apply_grad_mask: the registered gradient hooks
        self.anchor = {}    # the reference's default: no anchor, anchor_loss() returns zeros
        if track_anchor:    # GaussianModel's anchor bookkeeping (scene/gaussian_model.py:62-150)
            self._generation = torch.zeros(P, dtype=torch.int64, device=device)
            self._anchor_loss_schedule = torch.tensor([ANCHOR_WEIGHT_INIT_G0], dtype=torch.float32, device=device)
            self.update_anchor()
        self._make_optimizer()

    def update_anchor(self):
        """Snapshot the six parameters: the anchor the loss pulls them back to."""
        self.anchor = {a: getattr(self, a).detach().clone()
                       for a in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")}

    def update_anchor_loss_schedule(self):
        """After a densification: every generation's weight grows by the multiplier (capped), the generation born
        at the previous densification starts at the initial weight, and the one born now starts at 0."""
        s = torch.clamp_max(self._anchor_loss_schedule * ANCHOR_WEIGHT_MULTIPLIER, MAX_ANCHOR_WEIGHT)
        if s.numel() > 1:   # its last weight was 0 (the reference asserts it), so it multiplied to 0
            s[-1] = ANCHOR_WEIGHT_INIT
        self._anchor_loss_schedule = torch.cat([s, s.new_zeros(1)])

    def anchor_loss_torch(self):
        """GaussianModel.anchor_loss restated in plain torch (boolean indexing, so it synchronises with the host)."""
        out = {k: 0 for k in ANCHOR_LAMBDA}
        if not self.anchor:
            return out
        w = torch.gather(self._anchor_loss_schedule, 0, self._generation[self.mask])
        for key, value in self.anchor.items():
            delta = F.mse_loss(getattr(self, key)[self.mask], value[self.mask], reduction="none")
            delta = delta * w.view((-1,) + (1,) * (delta.dim() - 1))
            out[_ANCHOR_GROUP[key]] = out[_ANCHOR_GROUP[key]] + delta.mean()
        return out

    def apply_grad_mask(self):
        """GaussianEditor's ``apply_grad_mask`` (scene/gaussian_model.py:837-856): a hook on each parameter multiplies its
        gradient by ``mask``, read when the hook runs. Here on all six parameters, ``_rotation`` included (GaussianEditor
        leaves it out), so that every gradient of an unedited Gaussian is zero, as under ``render(..., grad_mask=...)``.
        Densification re-registers the hooks on the new tensors."""
        def hook(grad):
            return grad * (self.mask[:, None] if grad.ndim == 2 else self.mask[:, None, None])
        self.hooks = [getattr(self, a).register_hook(hook) for a in _SCENE_ATTR.values()]

    def _params(self):
        return [("xyz", self._xyz, 1.6e-5), ("f_dc", self._features_dc, 2.5e-3), ("f_rest", self._features_rest, 1.25e-4),
                ("opacity", self._opacity, 0.1), ("scaling", self._scaling, 1e-2), ("rotation", self._rotation, 2e-3)]

    def _make_optimizer(self):
        groups = [{"params": [p], "lr": lr, "name": n} for n, p, lr in self._params()]
        if self.optimizer_kind == "masked":   # built after every densification, so it always holds the current mask
            from .masked_adam import MaskedAdam
            self.optimizer = MaskedAdam(groups, eps=1e-15, capturable=self.capturable, mask=self.mask)
        elif self.capturable:
            self.optimizer = torch.optim.Adam(groups, eps=1e-15, capturable=True)
        else:
            self.optimizer = torch.optim.Adam(groups, eps=1e-15)

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

    def add_densification_stats_dense(self, viewspace_grad, update_filter):
        """add_densification_stats without boolean indexing (no host synchronisation, so it can be captured): the same
        values, since the rows outside the filter add exactly 0."""
        norm = torch.norm(viewspace_grad[:, :2], dim=-1, keepdim=True)
        self.xyz_gradient_accum.add_(torch.where(update_filter[:, None], norm, 0.0))
        self.denom.add_(update_filter[:, None].float())

    def densify_and_prune(self, max_densify_percent=0.01, min_opacity=0.005, masked=False):
        """Clone the `max_densify_percent` Gaussians with the largest mean view-space gradient, prune those below
        `min_opacity` (shape of scene/gaussian_model.py:768-809; the split branch is folded into clone). ``masked``: an
        edit under a gradient mask, whose unmasked view-space gradients are zeroed first (gaussian_model.py:773)."""
        with torch.no_grad():
            grads = (self.xyz_gradient_accum / self.denom.clamp_min(1)).squeeze(1)
            if masked:
                grads.masked_fill_(~self.mask, 0.0)
            P = grads.numel()
            k = max(1, int(P * max_densify_percent))
            sel = torch.topk(grads, k).indices
            keep = (torch.sigmoid(self._opacity).squeeze(1) >= min_opacity)
            keep[sel] = True
            kept = torch.nonzero(keep).squeeze(1)
            idx = torch.cat([kept, sel])
            for name in ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity"):
                setattr(self, name, getattr(self, name).detach()[idx].clone().requires_grad_(True))
            self.mask = self.mask[idx]
            n = idx.numel()
            dev = self._xyz.device
            self.max_radii2D = torch.zeros(n, device=dev)
            self.xyz_gradient_accum = torch.zeros(n, 1, device=dev)
            self.denom = torch.zeros(n, 1, device=dev)
            if self.anchor:   # clones are the new generation; then re-anchor and advance the schedule (:712-807)
                born = torch.full((sel.numel(),), self._anchor_loss_schedule.numel(), dtype=torch.int64, device=dev)
                self._generation = torch.cat([self._generation[kept], born])
                self.update_anchor()
                self.update_anchor_loss_schedule()
            self._make_optimizer()   # the reference re-stitches Adam state; the harness restarts it
        if self.hooks is not None:
            self.apply_grad_mask()


def make_view(cam: synth.Camera, device):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return SimpleNamespace(FoVx=2 * math.atan(cam.tanfovx), FoVy=2 * math.atan(cam.tanfovy),
                           image_height=cam.image_height, image_width=cam.image_width,
                           world_view_transform=t(cam.viewmatrix), full_proj_transform=t(cam.projmatrix),
                           camera_center=t(cam.campos))


def run_edit_loop(rasterizer_cls, steps=200, P=None, device="cuda", densification_interval=100, seed=0,
                  log=None, fused_activations=False, cuda_graph=False, static_capacity=False, deterministic=None,
                  grad_mask=None, optimizer="adam", semantic="render", semantic_log=None, anchor=None):
    """Returns a dict with total / render wall times (CUDA-event timed) and the per-step Gaussian counts.
    ``fused_activations`` renders the SH pass through ``render(..., fused_activations=True)`` (this repository's rasterizer only).
    ``cuda_graph=True`` captures one step per Gaussian count and replays it (see the module docstring);
    ``static_capacity=True`` runs that same step eagerly. Both size the rasterizer's static capacity as
    1.25 x the largest num_rendered over an eager pass of all views + 4096, recomputed after every densification, use
    Adam(capturable=True), and raise RuntimeError at the next densification point (or the end) if any forward
    exceeded the capacity. ``deterministic`` is passed to ``render`` when given.
    ``grad_mask`` trains under the scene's mask ("20 % nearest the origin") as a GaussianEditor edit does: ``"hooks"``
    registers ``EditScene.apply_grad_mask`` (GaussianEditor's hooks, on all six parameters), ``"kernel"`` passes
    ``grad_mask=scene.mask`` to the SH render instead; both zero the unmasked view-space gradients before densifying.
    ``None`` (default): no mask.
    ``optimizer``: ``"adam"`` (default) steps ``torch.optim.Adam``; ``"masked"`` steps ``MaskedAdam`` on the scene's
    mask (rebuilt with the new mask at every densification, inside the captured graph with ``cuda_graph``), which
    needs a ``grad_mask``.
    ``semantic``: where the step's semantic map (the mask drawn in white, thresholded) comes from. ``"render"``
    (default) renders it as GaussianEditor does, with a second forward ``render(..., override_color=mask)``;
    ``"fused"`` takes it from forward #1's ``mask_render`` output (``render(..., mask_render=scene.mask)``, this
    repository's rasterizer only): the same bits without the second forward.
    ``semantic_log``: None, or a list that receives every step's thresholded semantic map (bool [H,W]).
    ``anchor``: GaussianEditor's anchor loss. ``None`` (default) leaves it out. ``"torch"`` (``EditScene.anchor_loss_torch``,
    which synchronises: eager steps only) or ``"kernel"`` (``gaussianeditor_b200.anchor_loss``, capturable) adds
    ``sum(ANCHOR_LAMBDA[k] * loss[k])`` to every step's loss, with the scene tracking generations, anchors and the weight
    schedule across densifications; the result then also holds the final ``generation`` and ``anchor_schedule``."""
    from . import gaussian_renderer as GR
    if grad_mask not in (None, "hooks", "kernel"):
        raise ValueError(f'grad_mask must be None, "hooks" or "kernel", got {grad_mask!r}')
    if semantic not in ("render", "fused"):
        raise ValueError(f'semantic must be "render" or "fused", got {semantic!r}')
    if anchor not in (None, "torch", "kernel"):
        raise ValueError(f'anchor must be None, "torch" or "kernel", got {anchor!r}')
    _check_optimizer(optimizer, grad_mask)
    fixed = bool(cuda_graph or static_capacity)
    if anchor == "torch" and fixed:
        raise ValueError('anchor="torch" synchronises with the host (boolean indexing): it cannot run in the '
                         'static-capacity or CUDA-graph step; use anchor="kernel"')
    cloud, cams = synth.make_config("c5", P=P)
    scene = EditScene(cloud, device, capturable=fixed, optimizer=optimizer, track_anchor=anchor is not None)
    anchor_term = None
    if anchor is not None:
        from .anchor_loss import anchor_loss
        anchor_fn = scene.anchor_loss_torch if anchor == "torch" else (lambda: anchor_loss(scene))

        def anchor_term(loss):   # GassuianEditorEdit.training_step: loss += value * lambda, key by key
            for k, v in anchor_fn().items():
                loss = loss + v * ANCHOR_LAMBDA[k]
            return loss
    if grad_mask == "hooks":
        scene.apply_grad_mask()
    # the SH render's mask argument, looked up per step: densification replaces scene.mask
    mask_kw = (lambda: {"grad_mask": scene.mask}) if grad_mask == "kernel" else (lambda: {})
    fused_sem = semantic == "fused"
    if fused_sem:   # forward #1 also draws the mask
        mask_kw = (lambda kw=mask_kw: {**kw(), "mask_render": scene.mask})
    views = [make_view(c, device) for c in cams]
    pipe = SimpleNamespace(convert_SHs_python=False, compute_cov3D_python=False, debug=False)
    bg = torch.zeros(3, device=device)
    opt = {} if deterministic is None else {"deterministic": bool(deterministic)}
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
        if fixed:
            loop = _FixedCapacityStep(GR, scene, views, targets, pipe, bg, fused_activations, opt, cuda_graph, mask_kw,
                                      fused_sem, semantic_log is not None, anchor_term)
        render_ms = 0.0
        counts, losses, radii_trace = [], [], []
        rng = np.random.default_rng(seed)
        torch.cuda.synchronize()
        t_all0, t_all1 = ev(), ev()
        t_all0.record()
        pend = []
        for step in range(1, steps + 1):
            k = int(rng.integers(len(views)))
            if fixed:
                loss = loop.step(k)
                sem_map = loop.semantic
            else:
                e0, e1, e2, e3 = ev(), ev(), ev(), ev()
                e0.record()
                pkg = GR.render(views[k], scene, pipe, bg, fused_activations=fused_activations, **opt,
                                **mask_kw())                                                          # forward #1
                if fused_sem:
                    sem = pkg["mask_render"]
                else:
                    sem = GR.render(views[k], scene, pipe, bg,
                                    override_color=scene.mask[..., None].float().repeat(1, 3))["render"]  # forward #2
                e1.record()
                sem_map = torch.norm(sem, dim=0) > 0.8                                                # thresholded: no grad
                loss = 10.0 * (pkg["render"] - targets[k]).abs().mean() + 0.0 * sem_map.float().mean()
                if anchor_term is not None:
                    loss = anchor_term(loss)
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
            if semantic_log is not None:
                semantic_log.append(sem_map)
            if step % densification_interval == 0 and step < steps:
                if fixed:
                    loop.check_capacity()
                radii_trace.append(scene.max_radii2D.clone())   # what the reference's prune test reads (:790-795)
                scene.densify_and_prune(masked=grad_mask is not None)
                if fixed:
                    loop.reset()
            counts.append(scene._xyz.shape[0])
        t_all1.record()
        torch.cuda.synchronize()
        if fixed:
            loop.check_capacity()
        for e0, e1, e2, e3 in pend:   # backward time includes the few autograd elementwise kernels around it
            render_ms += e0.elapsed_time(e1) + e2.elapsed_time(e3)
        total_ms = t_all0.elapsed_time(t_all1)
    finally:
        GR.GaussianRasterizer = old
    out = dict(steps=steps, total_ms=total_ms, render_ms=render_ms, render_fraction=render_ms / total_ms,
               ms_per_step=total_ms / steps, P_first=counts[0], P_last=counts[-1], final_loss=float(loss.detach()),
               counts=counts, losses=torch.stack(losses).cpu().tolist(), max_radii2D=scene.max_radii2D.cpu(),
               max_radii2D_at_densify=[r.cpu() for r in radii_trace],
               params={n: getattr(scene, a).detach() for n, a in _SCENE_ATTR.items()}, optimizer=scene.optimizer,
               mask=scene.mask)
    if anchor is not None:
        out.update(generation=scene._generation, anchor_schedule=scene._anchor_loss_schedule)
    if fixed:   # the step is not split by events: no render time
        out.update(render_ms=None, render_fraction=None, capacities=loop.capacities)
    return out


def _check_optimizer(optimizer, grad_mask):
    if optimizer not in ("adam", "masked"):
        raise ValueError(f'optimizer must be "adam" or "masked", got {optimizer!r}')
    if optimizer == "masked" and grad_mask is None:
        raise ValueError('optimizer="masked" updates only the masked rows: it needs grad_mask="hooks" or "kernel"')


_SCENE_ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
               "scaling": "_scaling", "rotation": "_rotation"}   # EditScene's param-group names -> attributes


def sharded_scene(cloud: synth.Cloud, device, plan, optimizer="adam") -> EditScene:
    """The EditScene of the whole `cloud` (mask included) cut to `plan`'s rows, with zero statistics and a fresh
    optimizer (`optimizer` as in ``EditScene``)."""
    from .sharded import shard_slice
    scene = EditScene(cloud, device, optimizer=optimizer)
    with torch.no_grad():
        for attr in _SCENE_ATTR.values():
            setattr(scene, attr, shard_slice(getattr(scene, attr).detach(), plan).clone().requires_grad_(True))
        scene.mask = shard_slice(scene.mask, plan).clone()
        n = plan.count
        scene.max_radii2D = torch.zeros(n, device=device)
        scene.xyz_gradient_accum = torch.zeros(n, 1, device=device)
        scene.denom = torch.zeros(n, 1, device=device)
    scene._make_optimizer()
    return scene


def run_sharded_edit_loop(steps=200, P=None, densification_interval=100, seed=0, mode=None, deterministic=False,
                          group=None, max_densify_percent=0.01, min_opacity=0.005, grad_mask=None,
                          optimizer="adam"):
    """The config-5 step of ``run_edit_loop`` on a Gaussian-sharded cloud, one process per GPU (collective: every rank
    of `group` calls it with the same arguments; the process group must exist, NCCL).

    Every rank builds the same synthetic cloud and "20 % nearest the origin" mask and keeps its ``shard_slice``. Each
    step renders the same view on every rank through ``ShardedGaussianRasterizer`` (SH colours with gradient, then
    ``colors_precomp = mask``), takes the L1 loss on the full frame, back-propagates, updates ``max_radii2D`` and the
    densification statistics from the local radii and ``viewspace_points.grad``, and runs Adam on the local rows.
    Every `densification_interval` steps (not after the last): ``global_top_k`` of ``xyz_gradient_accum / denom`` picks
    the clone set, each rank prunes low opacity (keeping the selected rows) and appends its clones with
    ``optim_surgery`` (clones start with zero moments, kept rows keep theirs: the reference's behaviour), ``rebalance``
    with K = 2 moves rows, Adam state and the mask to their new owners, the statistics restart at zero and the
    rasterizer is re-created for the new size. `mode` and `deterministic` go to the rasterizer.
    ``grad_mask`` trains under the mask as ``run_edit_loop`` does: ``"hooks"`` registers ``EditScene.apply_grad_mask`` on
    the local rows (again after every densification, which swaps the parameters), ``"kernel"`` passes this rank's
    ``scene.mask`` to forward #1 (``ShardedGaussianRasterizer.forward(..., grad_mask=...)``); both zero the unmasked
    view-space statistics before ``global_top_k``. ``None`` (default): no mask. ``optimizer`` as in ``run_edit_loop``:
    ``"masked"`` steps ``MaskedAdam`` on this rank's mask, re-set to the mask ``rebalance`` carries after every
    densification.

    Returns ``run_edit_loop``'s dict (counts are global) plus ``densify`` (per densification: ms of selection, surgery,
    rebalance and re-creation, bytes moved across ranks), ``params`` (this rank's final rows), ``plan`` and ``mode``."""
    from .gaussian_renderer import _settings_for
    from .sharded import Exchange, ShardPlan, ShardedGaussianRasterizer
    if grad_mask not in (None, "hooks", "kernel"):
        raise ValueError(f'grad_mask must be None, "hooks" or "kernel", got {grad_mask!r}')
    _check_optimizer(optimizer, grad_mask)
    device = torch.device("cuda", torch.cuda.current_device())
    ex = Exchange(group)
    cloud, cams = synth.make_config("c5", P=P)
    plan = ShardPlan(cloud.means3D.shape[0], ex.world, ex.rank)
    scene = sharded_scene(cloud, device, plan, optimizer)
    if grad_mask == "hooks":
        scene.apply_grad_mask()
    views = [make_view(c, device) for c in cams]
    bg = torch.zeros(3, device=device)
    settings = lambda v: _settings_for(v, bg, 1.0, scene.active_sh_degree)
    make = lambda p: ShardedGaussianRasterizer(settings(views[0]), p.P_total, group=group, mode=mode,
                                               deterministic=bool(deterministic))
    rast = make(plan)
    mode = rast.mode

    def forward(view, colors=None, mask=None):
        rast.raster_settings = settings(view)
        means2D = torch.zeros_like(scene._xyz, requires_grad=True) + 0   # viewspace_points, as render() makes it
        if means2D.requires_grad:   # not under no_grad (the targets)
            means2D.retain_grad()
        kw = dict(shs=scene.get_features) if colors is None else dict(colors_precomp=colors)
        if mask is not None:
            kw["grad_mask"] = mask.contiguous()
        color, radii, _ = rast(means3D=scene.get_xyz, means2D=means2D, opacities=scene.get_opacity,
                               scales=scene.get_scaling, rotations=scene.get_rotation, **kw)
        return color, radii, means2D

    ev = lambda: torch.cuda.Event(enable_timing=True)
    try:
        with torch.no_grad():   # cached originals -> edited targets (guidance stub: + seeded noise), as run_edit_loop
            g = torch.Generator(device=device).manual_seed(seed)
            targets = []
            for v in views:
                img = forward(v)[0]
                targets.append((img + 0.05 * torch.randn(img.shape, generator=g, device=device)).clamp(0, 1))
        counts, losses, radii_trace, pend, densify = [], [], [], [], []
        rng = np.random.default_rng(seed)
        torch.cuda.synchronize()
        t_all0, t_all1 = ev(), ev()
        t_all0.record()
        for step in range(1, steps + 1):
            k = int(rng.integers(len(views)))
            e0, e1, e2, e3 = ev(), ev(), ev(), ev()
            e0.record()
            color, radii, means2D = forward(views[k], mask=scene.mask if grad_mask == "kernel" else None)  # #1
            sem, _, _ = forward(views[k], scene.mask[..., None].float().repeat(1, 3))          # forward #2
            e1.record()
            semantic = torch.norm(sem, dim=0) > 0.8
            loss = 10.0 * (color - targets[k]).abs().mean() + 0.0 * semantic.float().mean()
            scene.optimizer.zero_grad(set_to_none=True)
            e2.record()
            loss.backward()
            e3.record()
            pend.append((e0, e1, e2, e3))
            loss = loss.detach()   # the graph (and the workspaces its forwards hold) dies here, not at the next step
            del color, sem
            with torch.no_grad():
                vis = radii > 0
                scene.max_radii2D[vis] = torch.max(scene.max_radii2D[vis], radii[vis].float())
                scene.add_densification_stats(means2D.grad, vis)
            scene.optimizer.step()
            losses.append(loss.detach())
            if step % densification_interval == 0 and step < steps:
                radii_trace.append(scene.max_radii2D.clone())
                plan, phase = sharded_densify(scene, ex, plan, rast, max_densify_percent, min_opacity,
                                              masked=grad_mask is not None)
                if grad_mask == "hooks":
                    scene.apply_grad_mask()   # the new parameters take the hooks
                rast = make(plan)
                torch.cuda.synchronize()
                phase["recreate"] = (time.perf_counter() - phase.pop("_t")) * 1e3
                densify.append(phase)
            counts.append(plan.P_total)
        t_all1.record()
        torch.cuda.synchronize()
        render_ms = sum(e0.elapsed_time(e1) + e2.elapsed_time(e3) for e0, e1, e2, e3 in pend)
        total_ms = t_all0.elapsed_time(t_all1)
    finally:
        rast.close()
    return dict(steps=steps, total_ms=total_ms, render_ms=render_ms, render_fraction=render_ms / total_ms,
                ms_per_step=total_ms / steps, P_first=counts[0], P_last=counts[-1], final_loss=float(loss.detach()),
                counts=counts, losses=torch.stack(losses).cpu().tolist(), max_radii2D=scene.max_radii2D.cpu(),
                max_radii2D_at_densify=[r.cpu() for r in radii_trace], densify=densify, plan=plan, mode=mode,
                world=ex.world, params={n: getattr(scene, a).detach() for n, a in _SCENE_ATTR.items()},
                mask=scene.mask, optimizer=scene.optimizer)


def sharded_densify(scene, ex, plan, rast=None, max_densify_percent=0.01, min_opacity=0.005, masked=False):
    """One densification of run_sharded_edit_loop (collective) on this rank's rows of `scene`: global top-k, local prune
    and clone, rebalance (K = 2, the mask carried along), statistics reset; closes `rast`. Returns (new plan, phase
    times in ms and bytes moved); the caller re-creates the rasterizer and times that from ``phase["_t"]``. ``masked``:
    an edit under a gradient mask, whose unmasked view-space gradients are zeroed before the selection."""
    from . import optim_surgery
    from . import shard_rebalance as SR
    phase = {}
    torch.cuda.synchronize()
    marks = [time.perf_counter()]

    def lap(name):
        torch.cuda.synchronize()
        marks.append(time.perf_counter())
        phase[name] = (marks[-1] - marks[-2]) * 1e3

    with torch.no_grad():
        grads = (scene.xyz_gradient_accum / scene.denom).squeeze(1)     # NaN where denom == 0: counts as 0
        if masked:
            grads.masked_fill_(~scene.mask, 0.0)
        k = max(1, int(plan.P_total * max_densify_percent))
        sel = SR.global_top_k(ex, plan, grads, k)
        lap("select")
        keep = (torch.sigmoid(scene._opacity).squeeze(1) >= min_opacity) | sel
        kept = optim_surgery.prune_optimizer(scene.optimizer, keep)
        clone = sel[keep]
        optim_surgery.cat_tensors_to_optimizer(scene.optimizer, {n: p.detach()[clone] for n, p in kept.items()})
        mask = torch.cat((scene.mask[keep], scene.mask[sel]))
        counts = [int(keep.sum()), int(sel.sum())]
        lap("surgery")
        stats = {}
        new_plan, (scene.mask,) = SR.rebalance(ex, plan, counts, scene.optimizer, extras=(mask,), stats=stats)
        if scene.optimizer_kind == "masked":
            scene.optimizer.set_mask(scene.mask)
        for group in scene.optimizer.param_groups:
            setattr(scene, _SCENE_ATTR[group["name"]], group["params"][0])
        n = new_plan.count
        dev = scene._xyz.device
        scene.max_radii2D = torch.zeros(n, device=dev)
        scene.xyz_gradient_accum = torch.zeros(n, 1, device=dev)
        scene.denom = torch.zeros(n, 1, device=dev)
        lap("rebalance")
    phase.update(bytes_moved=stats["bytes_moved"], rows_moved=stats["rows_moved"], P_new=new_plan.P_total)
    if rast is not None:
        rast.close()
    phase["_t"] = marks[-1]
    return new_plan, phase


class _FixedCapacityStep:
    """One edit-loop step on the rasterizer's static-capacity forward, run eagerly or as a replayed CUDA graph.

    The capacity is sized once per Gaussian count (`reset`). With `cuda_graph`, the first step after a reset runs eagerly
    on a side stream (it creates Adam's state and warms every lazy initialisation), the second is captured, and every
    step copies its camera and target into the captured input tensors and replays. Overflows are accumulated on the
    device and read only by `check_capacity`. With `fused_semantic` the semantic map comes from forward #1's `mask_render`
    output (there is no forward #2); with `keep_semantic` each step leaves its own copy of the map in `semantic`.
    `anchor_term`, when given, adds the anchor loss to the step's loss (it must not synchronise)."""

    def __init__(self, GR, scene, views, targets, pipe, bg, fused_activations, opt, cuda_graph, mask_kw=dict,
                 fused_semantic=False, keep_semantic=False, anchor_term=None):
        self.GR, self.scene, self.views, self.targets, self.pipe, self.bg = GR, scene, views, targets, pipe, bg
        self.fused, self.opt, self.cuda_graph, self.mask_kw = fused_activations, opt, cuda_graph, mask_kw
        self.fused_semantic, self.keep_semantic, self.semantic = fused_semantic, keep_semantic, None
        self.anchor_term = anchor_term
        dev = bg.device
        self.overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        v0 = views[0]
        self.view = SimpleNamespace(**vars(v0))   # the captured camera: same intrinsics, pose tensors copied per step
        self.view.world_view_transform = v0.world_view_transform.clone()
        self.view.full_proj_transform = v0.full_proj_transform.clone()
        self.view.camera_center = v0.camera_center.clone()
        self.target = targets[0].clone()
        self.capacities = []
        self.reset()

    def reset(self):
        """New Gaussian count: size the capacity from an eager pass over all views, drop the captured graph."""
        from .rasterizer import _RasterizeGaussians
        r_max = 0
        with torch.no_grad():
            for v in self.views:
                self.GR.render(v, self.scene, self.pipe, self.bg)
                r_max = max(r_max, int(_RasterizeGaussians.last_state.num_rendered))
        self.capacity = int(r_max * 1.25) + 4096
        self.capacities.append(self.capacity)
        self.graph = self.captured = None
        self.warm = False

    def _body(self, view, target):
        GR, scene = self.GR, self.scene
        pkg = GR.render(view, scene, self.pipe, self.bg, fused_activations=self.fused, static_capacity=self.capacity,
                        **self.opt, **self.mask_kw())                                                 # forward #1
        if self.fused_semantic:   # forward #1's mask image: one status covers both
            sem_pkg, sem = None, pkg["mask_render"]
        else:
            sem_pkg = GR.render(view, scene, self.pipe, self.bg,
                                override_color=scene.mask[..., None].float().repeat(1, 3),
                                static_capacity=self.capacity, **self.opt)                             # forward #2
            sem = sem_pkg["render"]
        semantic = torch.norm(sem, dim=0) > 0.8
        self.semantic = semantic
        loss = 10.0 * (pkg["render"] - target).abs().mean() + 0.0 * semantic.float().mean()
        if self.anchor_term is not None:
            loss = self.anchor_term(loss)
        scene.optimizer.zero_grad(set_to_none=True)
        loss.backward()
        with torch.no_grad():
            vis = pkg["visibility_filter"]
            scene.max_radii2D.copy_(torch.where(vis, torch.maximum(scene.max_radii2D, pkg["radii"].float()),
                                                scene.max_radii2D))
            scene.add_densification_stats_dense(pkg["viewspace_points"].grad, vis)
            torch.maximum(self.overflow, pkg["status"][1:], out=self.overflow)
            if sem_pkg is not None:
                torch.maximum(self.overflow, sem_pkg["status"][1:], out=self.overflow)
        scene.optimizer.step()
        return loss.detach()

    def step(self, k):
        if not self.cuda_graph:
            return self._body(self.views[k], self.targets[k])
        if not self.warm:   # eager first step of this Gaussian count, on a side stream as torch.cuda.graph wants
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                loss = self._body(self.views[k], self.targets[k])
            torch.cuda.current_stream().wait_stream(side)
            self.warm = True
            return loss
        v = self.views[k]
        self.view.world_view_transform.copy_(v.world_view_transform)
        self.view.full_proj_transform.copy_(v.full_proj_transform)
        self.view.camera_center.copy_(v.camera_center)
        self.target.copy_(self.targets[k])
        if self.graph is None:
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.captured = self._body(self.view, self.target)
            self.captured_semantic = self.semantic
        self.graph.replay()
        if self.keep_semantic:   # the captured map is overwritten by the next replay
            self.semantic = self.captured_semantic.clone()
        return self.captured.clone()

    def check_capacity(self):
        """Synchronises: raises RuntimeError if any forward since the start exceeded its static capacity."""
        if int(self.overflow.item()):
            raise RuntimeError(f"a forward exceeded the static capacity {self.capacity}: its frame was rendered empty")
