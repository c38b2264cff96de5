"""Fixed-capacity forward on the Gaussian-sharded rasterizer, one process per GPU.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
      tools/sharded_static_bench.py [--config c4] [--P N] [--rounds 3] [--steps 10] [--warmup 3]

Config 4's cloud at 1920x1080, fwd + bwd of this rank's rows (colour loss) through ShardedGaussianRasterizer, for every
exchange (dense with NCCL, dense with peer stores, sparse; the last two need peer mappings):
  * default -- the host-sized path (waits for R once per forward)
  * static  -- static_capacity=N, called eagerly
  * graph   -- static_capacity=N, the step captured once in a CUDA graph and replayed
N = 1.25 x the largest per-rank R (all-reduce MAX) + 4096. The arms of one exchange are timed in alternated regions
(`rounds` of each) so that drift of the shared card falls on all alike; ms/step are means of the regions, max over
ranks. Prints the card name and its power limit, then ONE JSON line on rank 0.
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

from gaussianeditor_b200 import sharded as S, sparse_sharded as SS, synth  # noqa: E402
from sharded_apply_weights_bench import card, max_over_ranks, timed  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c4")
    ap.add_argument("--P", type=int, default=None)
    ap.add_argument("--rounds", type=int, default=3)
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
    leaves = {k: S.shard_slice(v, plan).contiguous().requires_grad_(True) for k, v in full.items()}
    m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
    cam = synth.ring_cameras(8, 4.5, 15.0, 1920, 1080, 61.0)[0]
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, dev)
    dL = torch.from_numpy(np.random.default_rng(3).random((3, 1080, 1920), dtype=np.float32)).to(dev)
    can_p2p = S.p2p_available(S.Exchange())
    settings = [("dense", False)] + ([("dense", True), ("sparse", True)] if can_p2p else [])
    card_name = card()
    out = dict(config=a.config, P=P, world=world, frame="1920x1080", card=card_name, results={})
    if rank == 0:
        print(f"card: {card_name}  world={world}  P={P}", flush=True)

    def step(m):
        def fn():
            for v in list(leaves.values()) + [m2]:
                v.grad = None
            (m(means2D=m2, **leaves)[0] * dL).sum().backward()
        return fn

    for mode, p2p in settings:
        default = S.ShardedGaussianRasterizer(rs, P, p2p=p2p, mode=mode)
        step(default)()
        torch.cuda.synchronize(dev)
        R = SS._SparseShardedRasterize.last["R"] if mode == "sparse" else S._ShardedRasterize.last_R
        N = int(1.25 * max_over_ranks(R, dev)) + 4096
        static = S.ShardedGaussianRasterizer(rs, P, p2p=p2p, mode=mode, static_capacity=N)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):              # warm-up: every scratch buffer is sized before the capture
            for _ in range(2):
                step(static)()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(dev)
        for v in list(leaves.values()) + [m2]:
            v.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            (static(means2D=m2, **leaves)[0] * dL).sum().backward()
        arms = dict(default=step(default), static=step(static), graph=graph.replay)
        acc = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                acc[k].append(timed(fn, a.steps, a.warmup, dev))
        static.check_capacity()
        key = f"{mode}{'-p2p' if (mode == 'dense' and p2p) else ''}"
        out["results"][key] = {k: round(max_over_ranks(float(np.mean(v)), dev), 3) for k, v in acc.items()}
        out["results"][key]["N"] = N
        if rank == 0:
            print(key, out["results"][key], flush=True)
        del graph
        torch.cuda.synchronize(dev)
        default.close()
        static.close()
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
