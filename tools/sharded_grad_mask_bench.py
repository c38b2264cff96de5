"""What ``ShardedGaussianRasterizer.forward(..., grad_mask=...)`` saves against GaussianEditor's hooks on a sharded cloud:
training step at BASELINE config 4 (5M Gaussians, SH degree 3, 1920x1080), dense and sparse, under three masks.

    python tools/sharded_grad_mask_bench.py [--P N] [--steps 10] [--regions 3] [--warmup 3]
    python -m torch.distributed.run --nproc-per-node N tools/sharded_grad_mask_bench.py ...   (more GPUs)

Without a launcher the script makes a one-rank NCCL group itself. Per mode and mask, two arms on the same cloud, cameras,
upstream image and warm-up, alternated region by region (the protocol of tools/grad_mask_bench.py):
  hooks  : ShardedGaussianRasterizer(rs, P, mode=...), the default backward, then a hook on each of this rank's five
           leaves multiplies its gradient by the rank's mask rows (GaussianEditor's apply_grad_mask, rotations included)
  kernel : the same module, forward(..., grad_mask=this rank's mask rows)
with loss = sum(colour * G). Masks: "20 % nearest the origin" (the edit harness's), the 5 % nearest, and all Gaussians
(there the "hooks" arm is the default backward alone). Each region times `--steps` forward + backward steps with CUDA
events (max over ranks); the line reports the median ms/step and the regions, and per step the render_bwd stage from
the library's "profile" option (it includes grad_mask_first) and grad_mask_first alone from torch.profiler, in separate
passes after the timed regions. The GPU name and power limit (NVML, read only) come from the same run. One JSON line on
rank 0.
"""
import argparse
import json
import os
import socket
import statistics
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gaussianeditor_b200 import _lib, sharded as S, synth  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402
from grad_mask_bench import power_limit_w  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=None)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--regions", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if "RANK" not in os.environ:
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        torch.cuda.set_device(0)
        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1,
                                device_id=torch.device("cuda", 0))
    else:
        os.environ.setdefault("LOCAL_WORLD_SIZE", os.environ.get("WORLD_SIZE", "1"))
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    dev = torch.device("cuda", torch.cuda.current_device())
    world, rank = dist.get_world_size(), dist.get_rank()
    cloud, cams = synth.make_config("c4", P=a.P)
    P = cloud.means3D.shape[0]
    plan = S.ShardPlan(P, world, rank)
    full = cloud_tensors(cloud, dev)
    loc = {k: S.shard_slice(v, plan).clone().requires_grad_(True) for k, v in full.items()}
    H, W = cams[0].image_height, cams[0].image_width
    G = torch.rand(3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    d = full["means3D"].norm(dim=1)
    q = lambda f: d <= d.kthvalue(max(1, int(f * P))).values
    masks = {"spatial20": q(0.2), "spatial5": q(0.05), "all": torch.ones(P, dtype=torch.bool, device=dev)}
    settings = [settings_from(c, (0, 0, 0), cloud.sh_degree, dev) for c in cams]
    del full
    out = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "world": world,
           "config4": f"P={P}, SH degree {cloud.sh_degree}, {W}x{H}", "steps_per_region": a.steps,
           "regions": a.regions}

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    for mode in ("dense", "sparse"):
        rast = S.ShardedGaussianRasterizer(settings[0], P, mode=mode)
        for mname, mfull in masks.items():
            mask = S.shard_slice(mfull, plan).contiguous()
            hooks = []

            def step(i, arm):
                for v in loc.values():
                    v.grad = None
                rast.raster_settings = settings[i % len(settings)]
                m2 = torch.zeros_like(loc["means3D"], requires_grad=True)
                color, _, _ = rast(means3D=loc["means3D"], means2D=m2, opacities=loc["opacities"], shs=loc["shs"],
                                   scales=loc["scales"], rotations=loc["rotations"],
                                   grad_mask=mask if arm == "kernel" else None)
                (color * G).sum().backward()

            def run(arm):
                if arm == "hooks" and mname != "all":
                    hooks[:] = [t.register_hook(lambda g: g * (mask[:, None] if g.ndim == 2 else mask[:, None, None]))
                                for t in loc.values()]
                for i in range(a.steps):
                    step(i, arm)
                for h in hooks:
                    h.remove()
                hooks.clear()

            arms = ("hooks", "kernel")
            for arm in arms:
                for _ in range(a.warmup):
                    run(arm)
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
            res["mask_fraction"] = float(mfull.float().mean())
            res["kernel_over_hooks"] = res["kernel"]["ms_per_step"] / res["hooks"]["ms_per_step"]
            out[f"{mode}_{mname}"] = res
        rast.close()
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
