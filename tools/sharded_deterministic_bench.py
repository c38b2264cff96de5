"""Cost of deterministic mode on the Gaussian-sharded rasterizer, one process per GPU.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
      tools/sharded_deterministic_bench.py [--config c4] [--P N] [--rounds 5] [--steps 5] [--warmup 2]

Config 4's cloud. For the dense and the sparse exchange (sparse needs peer mappings), ShardedGaussianRasterizer with
deterministic=True against the default:
  * fwd+bwd at 1920x1080 (config 4's frame), with the stage times of the library (render_bwd includes the
    deterministic reduction) and, in sparse mode, the phases between CUDA events;
  * one traced view (apply_weights, CH = 1) at 512x512 (config 5's tracing resolution).
The two settings are timed in alternated regions (`rounds` of each, default first) so that drift of the shared card
falls on both alike; the numbers are means per step / view of the regions, max over ranks. Also reports the
deterministic scratch of one step. Prints the card name and its power limit, then ONE JSON line on rank 0.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from gaussianeditor_b200 import _lib, sharded as S, sparse_sharded as SS, synth  # noqa: E402
from sharded_apply_weights_bench import card, max_over_ranks, timed  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c4")
    ap.add_argument("--P", type=int, default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    S.init_distributed("nccl", dev)
    cloud, _ = synth.make_config_cached(a.config, P=a.P)
    P = cloud.means3D.shape[0]
    full = cloud_tensors(cloud, dev)
    plan = S.ShardPlan(P, world, rank)
    loc = {k: S.shard_slice(v, plan).contiguous() for k, v in full.items()}
    cam_f = synth.ring_cameras(8, 4.5, 15.0, 1920, 1080, 61.0)[0]
    cam_t = synth.ring_cameras(8, 4.5, 15.0, 512, 512, 61.0)[1]
    rs_f = settings_from(cam_f, (0, 0, 0), cloud.sh_degree, dev)
    rs_t = settings_from(cam_t, (0, 0, 0), cloud.sh_degree, dev)
    dL = torch.from_numpy(np.random.default_rng(3).random((3, 1080, 1920), dtype=np.float32)).to(dev)
    yy, xx = torch.meshgrid(torch.arange(512, device=dev), torch.arange(512, device=dev), indexing="ij")
    iw = ((((xx - 256) ** 2 + (yy - 240) ** 2) < 150 ** 2).float())[None]
    leaves = {k: v.clone().requires_grad_(True) for k, v in loc.items()}
    m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
    w = torch.zeros(plan.count, 1, device=dev)
    c = torch.zeros(plan.count, 1, dtype=torch.int32, device=dev)
    lib = _lib.load()
    res = dict(card=card(), world=world, P=P, config=a.config, modes={})
    modes = ["dense"] + (["sparse"] if S.p2p_available(S.Exchange()) else [])
    for mode in modes:
        rasts = {det: S.ShardedGaussianRasterizer(rs_f, P, mode=mode, deterministic=det) for det in (False, True)}

        def step(r):
            r.raster_settings = rs_f
            color, _, _ = r(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], shs=leaves["shs"],
                            scales=leaves["scales"], rotations=leaves["rotations"])
            (color * dL).sum().backward()

        def trace(r):
            r.raster_settings = rs_t
            r.apply_weights(loc["means3D"], None, loc["opacities"], None, w, loc["scales"], loc["rotations"], None, c,
                            iw)

        out = {}
        for name, fn in (("fwd_bwd_1920x1080", step), ("trace_512x512", trace)):
            times = {False: [], True: []}
            for det in (False, True):
                timed(lambda: fn(rasts[det]), 1, a.warmup, dev)
            for _ in range(a.rounds):
                for det in (False, True):
                    times[det].append(timed(lambda: fn(rasts[det]), a.steps, 0, dev))
            out[name] = {("deterministic" if det else "default"): round(max_over_ranks(np.mean(t), dev), 3)
                         for det, t in times.items()}
        # stage split of one deterministic and one default step (library stage timers; sparse phases as CUDA events)
        for det in (False, True):
            _lib.set_option("profile", 1)
            _lib.profile_read()
            SS.TRACE = [] if mode == "sparse" else None
            step(rasts[det])
            torch.cuda.synchronize(dev)
            prof = _lib.profile_read()
            _lib.set_option("profile", 0)
            key = "deterministic" if det else "default"
            out[f"stages_{key}"] = {k: round(max_over_ranks(v[0], dev), 3) for k, v in prof.items()
                                    if k in ("render_bwd", "preprocess_bwd", "render_fwd")}
            if SS.TRACE:
                marks = SS.TRACE
                out[f"phases_{key}"] = {n: round(max_over_ranks(marks[i - 1][1].elapsed_time(e), dev), 3)
                                        for i, (n, e) in enumerate(marks) if i > 0}
            SS.TRACE = None
        R = int(S._ShardedRasterize.last_R) if mode == "dense" else int(SS._SparseShardedRasterize.last["R"])
        Pm = plan.P_pad if mode == "dense" else world * int(SS._SparseShardedRasterize.last["cap"])
        out["det_scratch_MB_rank0"] = round(lib.gsr_deterministic_scratch_bytes(Pm, R, 0) / 1e6, 1)
        res["modes"][mode] = out
        for r in rasts.values():
            r.close()
    if rank == 0:
        print(f"card: {res['card']}")
        print(json.dumps(res))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
