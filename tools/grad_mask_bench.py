"""What ``grad_mask`` saves against GaussianEditor's hooks: training step at BASELINE config 3 (1M Gaussians, 1600x1200)
under three masks, and the config-5 edit loop.

    python tools/grad_mask_bench.py [--steps 20] [--regions 3] [--warmup 5] [--loop-steps 200] [--loop-regions 2]

Config 3: per mask, two arms on the same cloud, cameras, upstream image and warm-up, alternated region by region:
  hooks  : GaussianRasterizer(rs), the default backward, then a hook on each of the five leaves multiplies its gradient
           by mask[:, None] (GaussianEditor's apply_grad_mask, rotations included)
  kernel : GaussianRasterizer(rs, grad_mask=mask)
with loss = sum(colour * G). Masks: the edit harness's "20 % nearest the origin", the 5 % nearest, and all Gaussians
(there the "hooks" arm is the default backward alone).
Each region times `--steps` forward + backward steps with CUDA events; the line reports the median ms/step, and per step
the render_bwd and preprocess_bwd stages from the library's "profile" option (render_bwd includes grad_mask_first) and
grad_mask_first alone from torch.profiler, in separate passes after the timed regions. `walked_edited` is the fraction of
the walked instances (positions below each tile's tile_last, summed over the tiles) whose Gaussian is masked.
Config 5: run_edit_loop for `--loop-steps` steps, grad_mask="hooks" against "kernel", eager and with cuda_graph=True,
alternated `--loop-regions` times; median ms/step. The GPU name and power limit (NVML, read only) come from the same run.
One JSON line.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gaussianeditor_b200 import _lib, synth  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians, forward_state_views  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402


def power_limit_w():
    try:
        import pynvml as nv
        nv.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "")
        idx = int(vis.split(",")[0]) if vis and vis.split(",")[0].strip().isdigit() else torch.cuda.current_device()
        return nv.nvmlDeviceGetPowerManagementLimit(nv.nvmlDeviceGetHandleByIndex(idx)) / 1000.0
    except Exception:
        return None


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def walked_edited(state, mask):
    v = forward_state_views(state)
    W, H = state.W, state.H
    gx, gy = (W + 15) // 16, (H + 15) // 16
    nc = torch.zeros(gy * 16, gx * 16, dtype=torch.int64, device=mask.device)
    nc[:H, :W] = v["n_contrib"].long()
    tl = nc.view(gy, 16, gx, 16).amax(dim=(1, 3)).reshape(-1)
    r = v["ranges"].long()
    n = torch.minimum(tl, (r[:, 1] - r[:, 0]).clamp_min(0))
    tile = torch.repeat_interleave(torch.arange(n.numel(), device=mask.device), (r[:, 1] - r[:, 0]).clamp_min(0))
    pos = torch.arange(tile.numel(), device=mask.device)
    start = r[:, 0][tile]
    walked = pos - start < n[tile]
    ids = v["point_list"].long()[: tile.numel()]
    return float((mask[ids] & walked).sum()) / max(float(walked.sum()), 1.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop-steps", type=int, default=200)
    ap.add_argument("--loop-regions", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda")
    out = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "steps_per_region": a.steps,
           "regions": a.regions}

    # ---- training step, config 3 ----
    cloud, cams = synth.make_config("c3")
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    H, W = cams[0].image_height, cams[0].image_width
    G = torch.rand(3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    d = ct["means3D"].detach().norm(dim=1)
    masks = {"spatial20": d <= torch.quantile(d, 0.2), "spatial5": d <= torch.quantile(d, 0.05),
             "all": torch.ones_like(d, dtype=torch.bool)}
    plain = [GaussianRasterizer(settings_from(c, (0, 0, 0), cloud.sh_degree, dev)) for c in cams]
    for mname, mask in masks.items():
        mk = [GaussianRasterizer(settings_from(c, (0, 0, 0), cloud.sh_degree, dev), grad_mask=mask) for c in cams]
        hooks = []

        def step(i, arm):
            for v in ct.values():
                v.grad = None
            m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
            r = (mk if arm == "kernel" else plain)[i % len(cams)]
            color, _, _ = r(means3D=ct["means3D"], means2D=m2, opacities=ct["opacities"], shs=ct["shs"],
                            scales=ct["scales"], rotations=ct["rotations"])
            (color * G).sum().backward()

        def run(arm):
            if arm == "hooks" and mname != "all":   # all ones: the hooks would multiply by 1, the default backward
                hooks[:] = [t.register_hook(lambda g: g * (mask[:, None] if g.ndim == 2 else mask[:, None, None]))
                            for t in ct.values()]
            for i in range(a.steps):
                step(i, arm)
            for h in hooks:
                h.remove()
            hooks.clear()

        arms = ("hooks", "kernel")
        for arm in arms:
            for _ in range(a.warmup):
                run(arm)
        torch.cuda.synchronize()
        times = {arm: [] for arm in arms}
        for _ in range(a.regions):
            for arm in arms:
                times[arm].append(timed(lambda: run(arm)) / a.steps)
        res = {}
        for arm in arms:
            _lib.set_option("profile", 1)
            _lib.profile_read()
            run(arm)
            prof = _lib.profile_read()
            _lib.set_option("profile", 0)
            res[arm] = {"ms_per_step": statistics.median(times[arm]), "regions": [round(t, 4) for t in times[arm]],
                        "render_bwd_ms": prof["render_bwd"][0] / a.steps,
                        "preprocess_bwd_ms": prof["preprocess_bwd"][0] / a.steps}
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
            run("kernel")
            torch.cuda.synchronize()
        first_us = sum(e.device_time_total for e in p.key_averages() if "grad_mask_first" in e.key)
        res["kernel"]["grad_mask_first_ms"] = first_us / 1e3 / a.steps
        step(0, "kernel")
        res["walked_edited"] = walked_edited(_RasterizeGaussians.last_state, mask)
        res["mask_fraction"] = float(mask.float().mean())
        res["kernel_over_hooks"] = res["kernel"]["ms_per_step"] / res["hooks"]["ms_per_step"]
        out[f"c3_{mname}"] = res
        del mk
    st = _RasterizeGaussians.last_state
    out["config3"] = f"P={cloud.means3D.shape[0]}, SH degree {cloud.sh_degree}, {W}x{H}, R={st.num_rendered}"
    del ct, plain, G
    torch.cuda.empty_cache()

    # ---- edit loop, config 5 ----
    from gaussianeditor_b200.edit_loop import run_edit_loop
    loop = {}
    for graph in (False, True):
        t = {"hooks": [], "kernel": []}
        for _ in range(a.loop_regions):
            for arm in t:
                r = run_edit_loop(GaussianRasterizer, steps=a.loop_steps, grad_mask=arm, cuda_graph=graph)
                t[arm].append(r["ms_per_step"])
        key = "cuda_graph" if graph else "eager"
        loop[key] = {arm: {"ms_per_step": statistics.median(v), "runs": [round(x, 4) for x in v]} for arm, v in t.items()}
        loop[key]["kernel_over_hooks"] = loop[key]["kernel"]["ms_per_step"] / loop[key]["hooks"]["ms_per_step"]
    out["c5_edit_loop"] = loop
    print(json.dumps(out))


if __name__ == "__main__":
    main()
