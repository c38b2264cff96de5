"""What the opt-in depth gradient costs per training step at BASELINE config 3 (1M Gaussians, 1600x1200).

    python tools/depth_grad_bench.py [--config c3] [--steps 20] [--regions 5] [--warmup 5]

Two arms on the same cloud, cameras, upstream images and warm-up, alternated region by region in one process:
  default : GaussianRasterizer(rs),                  loss = sum(colour * G)
  depth   : GaussianRasterizer(rs, depth_grad=True), loss = sum(colour * G) + sum(depth * G_D)
Each region times `--steps` forward + backward steps with CUDA events; the line reports the median ms/step over the
regions, and the render_bwd / preprocess_bwd stage times per step from the library's "profile" option (a separate
profiled pass per arm after the timed regions). The GPU name and its power limit (NVML, read only) are read in the
same run. Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gaussianeditor_b200 import _lib, synth  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer  # noqa: E402
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c3")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda")
    cloud, cams = synth.make_config(a.config)
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    H, W = cams[0].image_height, cams[0].image_width
    g = torch.Generator(device=dev).manual_seed(0)
    G = torch.rand(3, H, W, device=dev, generator=g)
    GD = torch.rand(1, H, W, device=dev, generator=g) - 0.5
    arms = {"default": [GaussianRasterizer(settings_from(c, (0, 0, 0), cloud.sh_degree, dev)) for c in cams],
            "depth": [GaussianRasterizer(settings_from(c, (0, 0, 0), cloud.sh_degree, dev), depth_grad=True)
                      for c in cams]}

    def step(i, arm):
        for v in ct.values():
            v.grad = None
        m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
        color, _, depth = arms[arm][i % len(cams)](means3D=ct["means3D"], means2D=m2, opacities=ct["opacities"],
                                                   shs=ct["shs"], scales=ct["scales"], rotations=ct["rotations"])
        loss = (color * G).sum()
        if arm == "depth":
            loss = loss + (depth * GD).sum()
        loss.backward()

    for arm in arms:
        for i in range(a.warmup):
            step(i, arm)
    torch.cuda.synchronize()
    times = {arm: [] for arm in arms}
    for _ in range(a.regions):
        for arm in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(a.steps):
                step(i, arm)
            e1.record()
            torch.cuda.synchronize()
            times[arm].append(e0.elapsed_time(e1) / a.steps)
    stages = {}
    for arm in arms:
        _lib.set_option("profile", 1)
        _lib.profile_read()
        for i in range(a.steps):
            step(i, arm)
        prof = _lib.profile_read()
        _lib.set_option("profile", 0)
        stages[arm] = {k: prof[k][0] / a.steps for k in ("render_bwd", "preprocess_bwd")}
    out = {"config": f"{a.config}: P={cloud.means3D.shape[0]}, SH degree {cloud.sh_degree}, {W}x{H}",
           "device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
           "steps_per_region": a.steps, "regions": a.regions}
    for arm in arms:
        out[f"{arm}_ms_per_step"] = statistics.median(times[arm])
        out[f"{arm}_ms_per_step_regions"] = [round(t, 4) for t in times[arm]]
        out[f"{arm}_render_bwd_ms"] = stages[arm]["render_bwd"]
        out[f"{arm}_preprocess_bwd_ms"] = stages[arm]["preprocess_bwd"]
    out["depth_over_default_ms"] = out["depth_ms_per_step"] - out["default_ms_per_step"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
