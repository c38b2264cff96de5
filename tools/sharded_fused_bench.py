"""Fused activations and the depth gradient on the Gaussian-sharded rasterizer, one process per GPU.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
      tools/sharded_fused_bench.py [--config c4] [--P N] [--rounds 3] [--steps 5] [--warmup 2]

Config 4's cloud at 1920x1080, fwd+bwd of this rank's rows through ShardedGaussianRasterizer, for every exchange
(dense with NCCL, dense with peer stores, sparse; the last two need peer mappings), with and without
deterministic=True:
  * act   -- the PyTorch activations of the rank's rows (sigmoid, exp, normalize, cat of the SH) + forward, colour loss
  * raw   -- forward_raw on the raw rows, colour loss
  * color -- depth_grad=True, activated forward, colour loss only (the depth gets no gradient)
  * depth -- depth_grad=True, activated forward, colour + depth loss
The variants of one setting are timed in alternated regions (`rounds` of each) so that drift of the shared card falls
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
import torch.nn.functional as F

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
    loc = {k: S.shard_slice(v, plan).contiguous() for k, v in full.items()}
    o = loc["opacities"].clamp(1e-6, 1 - 1e-6)
    raw = dict(means3D=loc["means3D"], opacity_logits=torch.log(o / (1 - o)),
               features_dc=loc["shs"][:, :1].contiguous(), features_rest=loc["shs"][:, 1:].contiguous(),
               log_scales=torch.log(loc["scales"]), raw_rotations=loc["rotations"] * 1.7)
    leaves = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
    cam = synth.ring_cameras(8, 4.5, 15.0, 1920, 1080, 61.0)[0]
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, dev)
    dL = torch.from_numpy(np.random.default_rng(3).random((3, 1080, 1920), dtype=np.float32)).to(dev)
    dD = torch.from_numpy(np.random.default_rng(4).random((1, 1080, 1920), dtype=np.float32)).to(dev) * 0.1
    can_p2p = S.p2p_available(S.Exchange())
    settings = [("dense", False)] + ([("dense", True), ("sparse", True)] if can_p2p else [])
    card_name = card()
    out = dict(config=a.config, P=P, world=world, frame="1920x1080", card=card_name, results={})
    if rank == 0:
        print(f"card: {card_name}  world={world}  P={P}", flush=True)

    def activated(lv):   # scene/gaussian_model.py's properties, on this rank's rows
        return dict(means3D=lv["means3D"], opacities=torch.sigmoid(lv["opacity_logits"]),
                    shs=torch.cat((lv["features_dc"], lv["features_rest"]), dim=1),
                    scales=torch.exp(lv["log_scales"]), rotations=F.normalize(lv["raw_rotations"]))

    for mode, p2p in settings:
        for det in (False, True):
            plain = S.ShardedGaussianRasterizer(rs, P, p2p=p2p, mode=mode, deterministic=det)
            dgrad = S.ShardedGaussianRasterizer(rs, P, p2p=p2p, mode=mode, deterministic=det, depth_grad=True)

            def act():
                color, _, _ = plain(means2D=m2, **activated(leaves))
                (color * dL).sum().backward()

            def fused():
                color, _, _ = plain.forward_raw(leaves["means3D"], m2, leaves["opacity_logits"], leaves["features_dc"],
                                                leaves["features_rest"], leaves["log_scales"], leaves["raw_rotations"])
                (color * dL).sum().backward()

            def color_only():
                color, _, _ = dgrad(means2D=m2, **activated(leaves))
                (color * dL).sum().backward()

            def color_depth():
                color, _, depth = dgrad(means2D=m2, **activated(leaves))
                ((color * dL).sum() + (depth * dD).sum()).backward()

            fns = dict(act=act, raw=fused, color=color_only, depth=color_depth)
            acc = {k: [] for k in fns}
            for _ in range(a.rounds):
                for k, fn in fns.items():
                    acc[k].append(timed(fn, a.steps, a.warmup, dev))
            key = f"{mode}{'-p2p' if (mode == 'dense' and p2p) else ''}{'-det' if det else ''}"
            out["results"][key] = {k: round(max_over_ranks(float(np.mean(v)), dev), 3) for k, v in acc.items()}
            if rank == 0:
                print(key, out["results"][key], flush=True)
            plain.close()
            dgrad.close()
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
