"""What deterministic mode costs: training step at BASELINE config 3 (1M Gaussians, 1600x1200) and apply_weights at
config 5 (500k Gaussians, 512x512), default against deterministic.

    python tools/deterministic_bench.py [--steps 20] [--regions 5] [--warmup 5] [--aw-views 48]

Step: two arms on the same cloud, cameras, upstream image and warm-up, alternated region by region in one process:
  default       : GaussianRasterizer(rs, deterministic=False)
  deterministic : GaussianRasterizer(rs, deterministic=True)
with loss = sum(colour * G). Each region times `--steps` forward + backward steps with CUDA events; the line reports
the median ms/step over the regions, and per step the render_bwd stage (which includes the deterministic reduction)
and preprocess_bwd from the library's "profile" option, in a separate profiled pass per arm after the timed regions.
apply_weights: one pass over `--aw-views` config-5 views per arm, alternated `--regions` times, median ms per call
(forward preprocess + binning + apply_weights, as the scene model calls it) and the apply_weights stage alone.
Memory: the deterministic scratch of one config-3 backward (gsr_deterministic_scratch_bytes) and the peak device memory
of one step in each arm. The GPU name and its power limit (NVML, read only) are read in the same run. One JSON line.
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
from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402

ARMS = {"default": False, "deterministic": True}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--aw-views", type=int, default=48)
    a = ap.parse_args()
    dev = torch.device("cuda")
    out = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "steps_per_region": a.steps,
           "regions": a.regions}

    # ---- training step, config 3 ----
    cloud, cams = synth.make_config("c3")
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    H, W = cams[0].image_height, cams[0].image_width
    G = torch.rand(3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    arms = {arm: [GaussianRasterizer(settings_from(c, (0, 0, 0), cloud.sh_degree, dev), deterministic=d) for c in cams]
            for arm, d in ARMS.items()}

    def step(i, arm):
        for v in ct.values():
            v.grad = None
        m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
        color, _, _ = arms[arm][i % len(cams)](means3D=ct["means3D"], means2D=m2, opacities=ct["opacities"],
                                              shs=ct["shs"], scales=ct["scales"], rotations=ct["rotations"])
        (color * G).sum().backward()

    def steps(arm):
        for i in range(a.steps):
            step(i, arm)

    for arm in arms:
        for i in range(a.warmup):
            step(i, arm)
    torch.cuda.synchronize()
    times = {arm: [] for arm in arms}
    for _ in range(a.regions):
        for arm in arms:
            times[arm].append(timed(lambda: steps(arm)) / a.steps)
    for arm in arms:
        _lib.set_option("profile", 1)
        _lib.profile_read()
        steps(arm)
        prof = _lib.profile_read()
        _lib.set_option("profile", 0)
        out[f"{arm}_ms_per_step"] = statistics.median(times[arm])
        out[f"{arm}_ms_per_step_regions"] = [round(t, 4) for t in times[arm]]
        out[f"{arm}_render_bwd_ms"] = prof["render_bwd"][0] / a.steps
        out[f"{arm}_preprocess_bwd_ms"] = prof["preprocess_bwd"][0] / a.steps
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        step(0, arm)
        torch.cuda.synchronize()
        out[f"{arm}_step_peak_mb"] = (torch.cuda.max_memory_allocated(dev) - base) / 2**20
    st = _RasterizeGaussians.last_state
    out["config3"] = f"P={cloud.means3D.shape[0]}, SH degree {cloud.sh_degree}, {W}x{H}, R={st.num_rendered}"
    out["deterministic_scratch_mb"] = _lib.load().gsr_deterministic_scratch_bytes(st.P, st.cap, 0) / 2**20
    out["deterministic_over_default"] = out["deterministic_ms_per_step"] / out["default_ms_per_step"]
    del ct, arms, G

    # ---- apply_weights, config 5 ----
    cloud, cams = synth.make_config("c5")
    cams = cams[:a.aw_views]
    ct = cloud_tensors(cloud, dev)
    P = cloud.means3D.shape[0]
    H, W = cams[0].image_height, cams[0].image_width
    iw = (torch.rand(1, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(1)) > 0.5).float()
    aw = {arm: [GaussianRasterizer(settings_from(c, (0, 0, 0), cloud.sh_degree, dev), deterministic=d) for c in cams]
          for arm, d in ARMS.items()}

    def pass_(arm):
        w = torch.zeros(P, 1, device=dev)
        cnt = torch.zeros(P, 1, dtype=torch.int32, device=dev)
        for r in aw[arm]:
            r.apply_weights(ct["means3D"], None, ct["opacities"], None, w, ct["scales"], ct["rotations"], None, cnt, iw)

    for arm in aw:
        pass_(arm)
    aw_times = {arm: [] for arm in aw}
    for _ in range(a.regions):
        for arm in aw:
            aw_times[arm].append(timed(lambda: pass_(arm)) / len(cams))
    for arm in aw:
        _lib.set_option("profile", 1)
        _lib.profile_read()
        pass_(arm)
        prof = _lib.profile_read()
        _lib.set_option("profile", 0)
        out[f"{arm}_apply_weights_call_ms"] = statistics.median(aw_times[arm])
        out[f"{arm}_apply_weights_stage_ms"] = prof["apply_weights"][0] / len(cams)
    out["config5"] = f"P={P}, {W}x{H}, {len(cams)} views"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
