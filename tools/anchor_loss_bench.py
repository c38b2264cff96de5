"""What ``anchor_loss`` saves against GaussianEditor's torch anchor loss: forward plus backward at BASELINE configs 3
and 5 under three masks, and the config-5 edit loop.

    python tools/anchor_loss_bench.py [--iters 50] [--regions 5] [--loop-steps 200] [--loop-regions 2]

Loss: the six GaussianEditor parameters of config 3 (1M Gaussians, SH degree 3) and config 5 (500k, degree 3), anchors
at a seeded offset, generations drawn from a three-generation schedule with one zero weight. Masks: all Gaussians, the
20 % and the 5 % nearest the origin. Three arms, each timed as training runs it, forward plus ``sum(lambda * loss)``
backward into ``.grad`` (set to None before each iteration): ``EditScene.anchor_loss_torch`` (the reference's
expression in plain torch), ``gaussianeditor_b200.anchor_loss`` run eagerly, and the same iteration captured once in a
CUDA graph and replayed (``kernel_graph``: no host overhead, so its time is the kernels' plus the few small torch
launches around them). Each region times `--iters` iterations with CUDA events; the arms alternate region by region
and the line reports the median ms per iteration.
Bytes model (host, from the mask), kernel arms: read the mask twice (P bytes each), the generations of the 32-byte
sectors holding an edited row twice, p and a of the sectors holding an edited element twice (forward and backward),
and write the six full gradients (4 * 59 * P bytes). Achieved bytes/s is model bytes over the median time, against
the H100 SXM's 3.35 TB/s of HBM3; it is reported for the kernel_graph arm.
Edit loop: run_edit_loop on config 5 with anchor="torch" against "kernel", eager; then the whole GaussianEditor step
captured (grad_mask="kernel", optimizer="masked", semantic="fused", cuda_graph=True) with anchor=None against
"kernel". Each pair alternates `--loop-regions` times; median ms/step. The GPU name and power limit (NVML, read only)
come from the same run. One JSON line.
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from masked_adam_bench import HBM_BYTES_PER_S, power_limit_w, sectors_touched, timed  # noqa: E402

from gaussianeditor_b200 import anchor_loss, synth  # noqa: E402
from gaussianeditor_b200.anchor_loss import KEYS, TERMS  # noqa: E402
from gaussianeditor_b200.edit_loop import ANCHOR_LAMBDA, EditScene  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer  # noqa: E402

SCHEDULE = [0.0169, 0.01, 0.0]


def kernel_bytes(mask: np.ndarray, Ds) -> int:
    P = mask.size
    b = 2 * P + 2 * 32 * sectors_touched(mask, 2)   # int64 generation = two floats per row
    b += sum(2 * 2 * 32 * sectors_touched(mask, D) for D in Ds if D)
    return b + 4 * sum(Ds) * P


def loss_step(cfg, a, dev):
    cloud, _ = synth.make_config(cfg)
    scene = EditScene(cloud, dev, track_anchor=True)
    P = scene._xyz.shape[0]
    gen = torch.Generator(device=dev).manual_seed(0)
    with torch.no_grad():
        for k in TERMS:   # the anchors stay, the parameters move away from them
            p = getattr(scene, k)
            p.add_(0.01 * torch.randn(p.shape, generator=gen, device=dev))
    scene._generation = torch.randint(0, len(SCHEDULE), (P,), generator=gen, device=dev)
    scene._anchor_loss_schedule = torch.tensor(SCHEDULE, device=dev)
    d = scene._xyz.detach().norm(dim=1)
    masks = {"all": torch.ones(P, dtype=torch.bool, device=dev), "spatial20": d <= torch.quantile(d, 0.2),
             "spatial5": d <= torch.quantile(d, 0.05)}
    Ds = [int(np.prod(getattr(scene, k).shape[1:])) for k in TERMS]
    out = {"P": P}

    def it(fn):
        for k in TERMS:
            getattr(scene, k).grad = None
        res = fn()
        loss = 0
        for k in KEYS:
            loss = loss + res[k] * ANCHOR_LAMBDA[k]
        loss.backward()

    kernel = lambda: anchor_loss(scene)
    for mname, mask in masks.items():
        scene.mask = mask
        arms = {"torch": scene.anchor_loss_torch, "kernel": kernel}
        vals = {}
        for arm, fn in arms.items():   # warm-up, and the two arms' values for the line
            for _ in range(3):
                it(fn)
            vals[arm] = [float(v) for v in fn().values()]
        side = torch.cuda.Stream()   # warm-up on a side stream, then capture one kernel iteration
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            it(kernel)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            it(kernel)
        arms["kernel_graph"] = None
        torch.cuda.synchronize()
        times = {arm: [] for arm in arms}
        for _ in range(a.regions):
            for arm, fn in arms.items():
                def run(fn=fn):
                    for _ in range(a.iters):
                        if fn is None:
                            graph.replay()
                        else:
                            it(fn)
                times[arm].append(timed(run) / a.iters)
        mb = kernel_bytes(mask.cpu().numpy(), Ds)
        res = {"mask_fraction": float(mask.float().mean()), "kernel_model_bytes": mb,
               "values": vals}
        for arm, t in times.items():
            res[arm] = {"ms_per_iter": statistics.median(t), "regions": [round(x, 4) for x in t]}
        kg = res["kernel_graph"]
        kg["achieved_TBps"] = mb / (kg["ms_per_iter"] * 1e-3) / 1e12
        kg["share_of_3.35TBps"] = mb / (kg["ms_per_iter"] * 1e-3) / HBM_BYTES_PER_S
        res["kernel_over_torch"] = res["kernel"]["ms_per_iter"] / res["torch"]["ms_per_iter"]
        out[mname] = res
        del graph
    del scene
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--loop-steps", type=int, default=200)
    ap.add_argument("--loop-regions", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda")
    out = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "iters_per_region": a.iters,
           "regions": a.regions}
    for cfg in ("c3", "c5"):
        out[f"loss_{cfg}"] = loss_step(cfg, a, dev)

    from gaussianeditor_b200.edit_loop import run_edit_loop
    captured = dict(grad_mask="kernel", optimizer="masked", semantic="fused", cuda_graph=True)
    loop = {}
    for key, arms in (("eager", {"torch": ("torch", {}), "kernel": ("kernel", {})}),
                      ("captured", {"none": (None, captured), "kernel": ("kernel", captured)})):
        t = {arm: [] for arm in arms}
        for _ in range(a.loop_regions):
            for arm, (anchor, kw) in arms.items():
                r = run_edit_loop(GaussianRasterizer, steps=a.loop_steps, anchor=anchor, **kw)
                t[arm].append(r["ms_per_step"])
        loop[key] = {arm: {"ms_per_step": statistics.median(v), "runs": [round(x, 4) for x in v]} for arm, v in t.items()}
    loop["eager"]["kernel_over_torch"] = loop["eager"]["kernel"]["ms_per_step"] / loop["eager"]["torch"]["ms_per_step"]
    out["c5_edit_loop"] = loop
    print(json.dumps(out))


if __name__ == "__main__":
    main()
