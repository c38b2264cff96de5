"""What the fixed-capacity forward saves: ms per step of three variants, alternated region by region in one process.

    python tools/static_capacity_bench.py [--steps 20] [--regions 3] [--warmup 3] [--loop-steps 200]

Variants:
  default : GaussianRasterizer as is (the host waits for num_rendered in every forward)
  static  : GaussianRasterizer(static_capacity=cap), eager (no host wait, no pinned word)
  graph   : the same step captured once with torch.cuda.graph and replayed, camera copied into the captured tensors
Config 3 (1M Gaussians, 1600x1200, 8 ring cameras): one forward + backward of loss = sum(colour * G) per step; the
capacity is 1.25 x the largest num_rendered over the cameras + 4096. Each region times `--steps` steps with CUDA events.
Config 5 (the edit loop of edit_loop.py: 500k Gaussians, 512x512, two forwards + one backward + densification stats +
Adam per step, densification every 100 steps): one `run_edit_loop` of `--loop-steps` steps per variant and region,
ms/step as the loop reports it (CUDA events around all steps, densification, capacity sizing and re-capture included).
default uses the harness's Adam; static and graph use Adam(capturable=True).
The lines report the median over the regions. The GPU name and its power limit (NVML, read only) are read in the same
run. One JSON line.
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
from gaussianeditor_b200 import synth  # noqa: E402
from gaussianeditor_b200.edit_loop import run_edit_loop  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402

ARMS = ("default", "static", "graph")


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


def config3(a, dev, out):
    cloud, cams = synth.make_config("c3")
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    H, W = cams[0].image_height, cams[0].image_width
    G = torch.rand(3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    settings = [settings_from(c, (0, 0, 0), cloud.sh_degree, dev) for c in cams]

    def run(rast):
        for v in ct.values():
            v.grad = None
        m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
        color, _, _ = rast(means3D=ct["means3D"], means2D=m2, opacities=ct["opacities"], shs=ct["shs"],
                           scales=ct["scales"], rotations=ct["rotations"])
        (color * G).sum().backward()

    default = [GaussianRasterizer(rs) for rs in settings]
    r_max = 0
    for r in default:
        run(r)
        r_max = max(r_max, _RasterizeGaussians.last_state.num_rendered)
    cap = int(r_max * 1.25) + 4096
    static = [GaussianRasterizer(rs, static_capacity=cap) for rs in settings]
    rs0 = settings[0]
    cam_t = rs0._replace(viewmatrix=rs0.viewmatrix.clone(), projmatrix=rs0.projmatrix.clone(),
                         campos=rs0.campos.clone())
    captured = GaussianRasterizer(cam_t, static_capacity=cap)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run(captured)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run(captured)

    def replay(i):
        rs = settings[i]
        cam_t.viewmatrix.copy_(rs.viewmatrix); cam_t.projmatrix.copy_(rs.projmatrix); cam_t.campos.copy_(rs.campos)
        graph.replay()

    step = {"default": lambda i: run(default[i % len(cams)]), "static": lambda i: run(static[i % len(cams)]),
            "graph": lambda i: replay(i % len(cams))}
    for arm in ARMS:
        for i in range(a.warmup):
            step[arm](i)
    torch.cuda.synchronize()
    times = {arm: [] for arm in ARMS}
    for _ in range(a.regions):
        for arm in ARMS:
            times[arm].append(timed(lambda: [step[arm](i) for i in range(a.steps)]) / a.steps)
    for arm in ARMS:
        out[f"c3_{arm}_ms_per_step"] = statistics.median(times[arm])
        out[f"c3_{arm}_ms_per_step_regions"] = [round(t, 4) for t in times[arm]]
    captured.check_capacity()
    out["c3"] = f"P={cloud.means3D.shape[0]}, SH degree {cloud.sh_degree}, {W}x{H}, max R={r_max}, capacity={cap}"


def config5(a, out):
    kw = {"default": {}, "static": {"static_capacity": True}, "graph": {"cuda_graph": True}}
    times = {arm: [] for arm in ARMS}
    counts = {}
    for _ in range(a.regions):
        for arm in ARMS:
            r = run_edit_loop(GaussianRasterizer, steps=a.loop_steps, **kw[arm])
            times[arm].append(r["ms_per_step"])
            counts[arm] = (r["P_first"], r["P_last"])
    for arm in ARMS:
        out[f"c5_{arm}_ms_per_step"] = statistics.median(times[arm])
        out[f"c5_{arm}_ms_per_step_regions"] = [round(t, 4) for t in times[arm]]
    out["c5"] = f"{a.loop_steps} steps, P first/last {counts['graph']}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--regions", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loop-steps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("static_capacity_bench.py needs a CUDA device")
    dev = torch.device("cuda")
    out = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "regions": a.regions}
    config3(a, dev, out)
    torch.cuda.empty_cache()
    config5(a, out)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
