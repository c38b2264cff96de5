"""Cost of one view of semantic tracing (apply_weights) on a sharded cloud, one process per GPU.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
      tools/sharded_apply_weights_bench.py [--config c4] [--P N] [--sizes 512x512,1920x1080] [--steps 10] [--warmup 3]

For each frame size (config 4's cloud; 512x512 is config 5's tracing resolution, 1920x1080 config 4's frame):
  * the single-GPU GaussianRasterizer.apply_weights on the whole cloud (rank 0);
  * ShardedGaussianRasterizer.apply_weights, sparse (needs peer mappings) and dense, on N ranks, with the sparse phases
    (preprocess+push, order, walk, return+barrier, gather: CUDA events between them) and the dense stages (library
    stage timers);
  * the sharded forward at the same view, for scale.
Times are CUDA events on the compute stream, mean per view, max over ranks. Prints the card name and its power limit,
then ONE JSON line on rank 0.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gaussianeditor_b200 import _lib, sharded as S, sparse_sharded as SS, synth  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        q = ""
    return q or torch.cuda.get_device_name()


def timed(fn, steps, warmup, dev):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize(dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize(dev)
    return a.elapsed_time(b) / steps


def max_over_ranks(x, dev):
    t = torch.tensor([float(x)], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c4")
    ap.add_argument("--P", type=int, default=None)
    ap.add_argument("--sizes", default="512x512,1920x1080")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    S.init_distributed("nccl", dev)
    cloud, _ = synth.make_config_cached(a.config, P=a.P)
    P = cloud.means3D.shape[0]
    full = cloud_tensors(cloud, dev)
    plan = S.ShardPlan(P, world, rank)
    loc = {k: S.shard_slice(v, plan).contiguous() for k, v in full.items()}
    res = dict(card=card(), world=world, P=P, config=a.config, sizes={})
    rasts = {}
    for size in a.sizes.split(","):
        W, H = (int(v) for v in size.split("x"))
        cam = synth.ring_cameras(8, 4.5, 15.0, W, H, 61.0)[0]
        rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, dev)
        yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
        iw = ((((xx - W / 2) ** 2 + (yy - H / 2) ** 2) < (0.3 * min(W, H)) ** 2).float())[None]
        out = {}
        if rank == 0:
            w = torch.zeros(P, 1, device=dev); c = torch.zeros(P, 1, dtype=torch.int32, device=dev)
            single = GaussianRasterizer(rs)
            out["single_gpu_ms"] = timed(lambda: single.apply_weights(full["means3D"], None, full["opacities"], None, w,
                                                                      full["scales"], full["rotations"], None, c, iw),
                                         a.steps, a.warmup, dev)
            del w, c
            torch.cuda.empty_cache()
        dist.barrier()
        w = torch.zeros(plan.count, 1, device=dev); c = torch.zeros(plan.count, 1, dtype=torch.int32, device=dev)
        for mode in ("sparse", "dense"):
            key = mode
            if key not in rasts:
                try:
                    rasts[key] = S.ShardedGaussianRasterizer(rs, P, mode=mode)
                except RuntimeError as e:   # sparse needs peer mappings
                    out[f"{mode}_error"] = str(e)
                    continue
            rast = rasts[key]
            rast.raster_settings = rs
            call = lambda: rast.apply_weights(loc["means3D"], None, loc["opacities"], None, w, loc["scales"],
                                              loc["rotations"], None, c, iw)
            out[f"{mode}_ms"] = max_over_ranks(timed(call, a.steps, a.warmup, dev), dev)
            # per-phase breakdown
            if mode == "sparse":
                sums = {}
                for _ in range(a.steps):
                    SS.TRACE = []
                    call()
                    torch.cuda.synchronize(dev)
                    marks = SS.TRACE
                    SS.TRACE = None
                    for (_, e0), (name, e1) in zip(marks, marks[1:]):
                        sums[name] = sums.get(name, 0.0) + e0.elapsed_time(e1)
                out["sparse_phases_ms"] = {k: max_over_ranks(v / a.steps, dev) for k, v in sums.items()}
            else:
                _lib.profile_read()
                _lib.set_option("profile", 1)
                for _ in range(a.steps):
                    call()
                _lib.set_option("profile", 0)
                prof = _lib.profile_read()
                out["dense_stages_ms"] = {k: max_over_ranks(v[0] / a.steps, dev) for k, v in prof.items() if v[1]}
            m2 = torch.zeros_like(loc["means3D"])
            with torch.no_grad():
                fwd = lambda: rast(means3D=loc["means3D"], means2D=m2, opacities=loc["opacities"], shs=loc["shs"],
                                   scales=loc["scales"], rotations=loc["rotations"])
                if mode == "sparse":
                    rk0 = rast.sparse_pool.all[0]
                    if (rk0.W, rk0.H) != (W, H):   # the sparse forward's frame size is fixed at construction
                        out["sparse_forward_ms"] = None
                        continue
                out[f"{mode}_forward_ms"] = max_over_ranks(timed(fwd, a.steps, a.warmup, dev), dev)
        res["sizes"][size] = out
    for r in rasts.values():
        r.close()
    if rank == 0:
        print(f"card: {res['card']}  world={world}  P={P}")
        print(json.dumps(res))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
