"""Alpha image and camera gradients on the Gaussian-sharded rasterizer, one process per GPU.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
      tools/sharded_alpha_camera_bench.py [--config c4] [--P N] [--rounds 3] [--steps 5] [--warmup 2]

Config 4's cloud at 1920x1080, fwd+bwd of this rank's rows through ShardedGaussianRasterizer, for every exchange
(dense with NCCL, dense with peer stores, sparse; the last two need peer mappings):
  * default -- both flags off, colour loss
  * alpha   -- return_alpha=True, colour + alpha loss
  * camera  -- camera_grad=True, colour loss (the camera arrays get their gradients)
  * both    -- return_alpha=True and camera_grad=True, colour + alpha loss
The variants of one exchange are timed in alternated regions (`rounds` of each) so that drift of the shared card falls
on all alike; ms/step are means of the regions, max over ranks. Prints the card name and its power limit, then ONE
JSON line on rank 0.
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

from gaussianeditor_b200 import sharded as S, synth  # noqa: E402
from sharded_apply_weights_bench import card, max_over_ranks, timed  # noqa: E402
from util import cloud_tensors, settings_from  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c4")
    ap.add_argument("--P", type=int, default=None)
    ap.add_argument("--rounds", type=int, default=3)
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
    leaves = {k: S.shard_slice(v, plan).contiguous().requires_grad_(True) for k, v in full.items()}
    m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
    cam = synth.ring_cameras(8, 4.5, 15.0, 1920, 1080, 61.0)[0]
    base = settings_from(cam, (0, 0, 0), cloud.sh_degree, dev)
    cam_rs = base._replace(**{k: getattr(base, k).clone().requires_grad_(True)
                              for k in ("viewmatrix", "projmatrix", "campos")})
    dL = torch.from_numpy(np.random.default_rng(3).random((3, 1080, 1920), dtype=np.float32)).to(dev)
    dA = torch.from_numpy(np.random.default_rng(4).random((1, 1080, 1920), dtype=np.float32)).to(dev) - 0.5
    can_p2p = S.p2p_available(S.Exchange())
    settings = [("dense", False)] + ([("dense", True), ("sparse", True)] if can_p2p else [])
    card_name = card()
    out = dict(config=a.config, P=P, world=world, frame="1920x1080", card=card_name, results={})
    if rank == 0:
        print(f"card: {card_name}  world={world}  P={P}", flush=True)

    for mode, p2p in settings:
        mods = dict(default=S.ShardedGaussianRasterizer(base, P, p2p=p2p, mode=mode),
                    alpha=S.ShardedGaussianRasterizer(base, P, p2p=p2p, mode=mode, return_alpha=True),
                    camera=S.ShardedGaussianRasterizer(cam_rs, P, p2p=p2p, mode=mode, camera_grad=True),
                    both=S.ShardedGaussianRasterizer(cam_rs, P, p2p=p2p, mode=mode, return_alpha=True,
                                                     camera_grad=True))

        def step(m):
            def fn():
                out = m(means2D=m2, **leaves)
                loss = (out[0] * dL).sum()
                if m.return_alpha:
                    loss = loss + (out[3] * dA).sum()
                loss.backward()
            return fn

        acc = {k: [] for k in mods}
        for _ in range(a.rounds):
            for k, m in mods.items():
                acc[k].append(timed(step(m), a.steps, a.warmup, dev))
        key = f"{mode}{'-p2p' if (mode == 'dense' and p2p) else ''}"
        out["results"][key] = {k: round(max_over_ranks(float(np.mean(v)), dev), 3) for k, v in acc.items()}
        if rank == 0:
            print(key, out["results"][key], flush=True)
        for m in mods.values():
            m.close()
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
