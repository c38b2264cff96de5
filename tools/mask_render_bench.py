"""What ``mask_render`` costs and saves: GaussianEditor's semantic map from the colour pass instead of a second forward.

    python tools/mask_render_bench.py [--steps 20] [--regions 5] [--warmup 5] [--loop-steps 100] [--loop-regions 3]

Config 3 (BASELINE: 1M Gaussians, SH degree 3, 1600x1200), forward only, three arms on the same cloud, cameras and
mask ("20 % nearest the origin"), alternated region by region after a warm-up of each:
  fwd1        : the colour forward alone
  fwd1+fwd2   : the colour forward, then GaussianEditor's second forward (colors_precomp = mask in three channels)
  fwd1_mask   : the colour forward with mask_render=mask (one forward that also writes the mask image)
Each region times `--steps` forwards per arm with CUDA events; the line reports the median ms per forward step, every
region, and the peak device memory of one step of each arm (torch.cuda.max_memory_allocated over the step, minus what
was allocated before it). `extra_ms` = fwd1_mask - fwd1 (the cost of the extra channel), `saved_ms` = fwd1+fwd2 -
fwd1_mask.
Config 5: run_edit_loop under grad_mask="kernel" and deterministic=False, semantic="render" (two forwards per step)
against "fused", eager and with cuda_graph=True, alternated `--loop-regions` times; median ms/step, every run, and the
peak device memory of each arm's run. The GPU name, power limit and SM clocks (nvidia-smi, read only) come from the
same run. One JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gaussianeditor_b200 import synth  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402


def gpu_info():
    """power limit and SM clocks of the device, read with nvidia-smi (no setting is changed)."""
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "")
        idx = vis.split(",")[0].strip() if vis and vis.split(",")[0].strip().isdigit() else str(torch.cuda.current_device())
        line = subprocess.run(["nvidia-smi", "-i", idx, f"--query-gpu={q}", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [v.strip() for v in line.split(",")]))
    except Exception:
        return None


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop-steps", type=int, default=100)
    ap.add_argument("--loop-regions", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda")
    out = {"device": torch.cuda.get_device_name(dev), "gpu_before": gpu_info(), "steps_per_region": a.steps,
           "regions": a.regions}

    # ---- forward only, config 3 ----
    cloud, cams = synth.make_config("c3")
    ct = cloud_tensors(cloud, dev, requires_grad=True)   # as in training: the second forward keeps its workspaces
    d = ct["means3D"].detach().norm(dim=1)
    mask = d <= torch.quantile(d, 0.2)
    white = mask.float()[:, None].repeat(1, 3)
    plain = [GaussianRasterizer(settings_from(c, (0, 0, 0), cloud.sh_degree, dev)) for c in cams]
    fused = [GaussianRasterizer(settings_from(c, (0, 0, 0), cloud.sh_degree, dev), mask_render=mask) for c in cams]
    geo = dict(opacities=ct["opacities"], scales=ct["scales"], rotations=ct["rotations"])

    def step(i, arm):
        m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
        k = i % len(cams)
        r = (fused if arm == "fwd1_mask" else plain)[k]
        outs = r(means3D=ct["means3D"], means2D=m2, shs=ct["shs"], **geo)
        sem = outs[-1] if arm == "fwd1_mask" else None
        if arm == "fwd1+fwd2":
            sem = plain[k](means3D=ct["means3D"], means2D=m2, colors_precomp=white, **geo)[0]
        return outs, sem

    def run(arm):
        for i in range(a.steps):
            step(i, arm)

    arms = ("fwd1", "fwd1+fwd2", "fwd1_mask")
    for arm in arms:
        for _ in range(a.warmup):
            run(arm)
    torch.cuda.synchronize()
    times = {arm: [] for arm in arms}
    for _ in range(a.regions):
        for arm in arms:
            times[arm].append(timed(lambda: run(arm)) / a.steps)
    c3 = {arm: {"ms": statistics.median(times[arm]), "regions": [round(t, 4) for t in times[arm]],
                "spread_ms": round(max(times[arm]) - min(times[arm]), 4),
                "peak_mib": round(peak_bytes(lambda: step(0, arm)) / 2 ** 20, 1)} for arm in arms}
    c3["extra_ms"] = c3["fwd1_mask"]["ms"] - c3["fwd1"]["ms"]
    c3["saved_ms"] = c3["fwd1+fwd2"]["ms"] - c3["fwd1_mask"]["ms"]
    step(0, "fwd1")
    st = _RasterizeGaussians.last_state
    H, W = cams[0].image_height, cams[0].image_width
    c3["config"] = f"P={cloud.means3D.shape[0]}, SH degree {cloud.sh_degree}, {W}x{H}, R={st.num_rendered}"
    out["c3_forward"] = c3
    del ct, plain, fused, white, mask, geo, st
    _RasterizeGaussians.last_state = None
    torch.cuda.empty_cache()

    # ---- edit loop, config 5 ----
    from gaussianeditor_b200.edit_loop import run_edit_loop
    loop = {}
    for graph in (False, True):
        t = {"render": [], "fused": []}
        peak = {}
        for _ in range(a.loop_regions):
            for arm in t:
                res = {}
                p = peak_bytes(lambda: res.update(run_edit_loop(GaussianRasterizer, steps=a.loop_steps,
                                                                grad_mask="kernel", cuda_graph=graph, semantic=arm)))
                t[arm].append(res["ms_per_step"])
                peak[arm] = max(peak.get(arm, 0), p)
                del res
                torch.cuda.empty_cache()
        key = "cuda_graph" if graph else "eager"
        loop[key] = {arm: {"ms_per_step": statistics.median(v), "runs": [round(x, 4) for x in v],
                           "peak_mib": round(peak[arm] / 2 ** 20, 1)} for arm, v in t.items()}
        loop[key]["fused_over_render"] = loop[key]["fused"]["ms_per_step"] / loop[key]["render"]["ms_per_step"]
    out["c5_edit_loop"] = loop
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
