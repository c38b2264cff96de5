"""What ``MaskedAdam`` saves against torch's Adam: the optimizer step alone at BASELINE configs 3 and 5, under three
masks, and the config-5 edit loop.

    python tools/masked_adam_bench.py [--steps 50] [--regions 5] [--warmup 10] [--loop-steps 200] [--loop-regions 2]

Optimizer step: the six GaussianEditor groups (xyz 3, f_dc 3, f_rest 45, opacity 1, scaling 3, rotation 4 floats per
Gaussian; lrs of EditScene, eps 1e-15) of config 3 (1M Gaussians, SH degree 3) and config 5 (500k, degree 3). Masks:
all Gaussians, the 20 % and the 5 % nearest the origin. Gradients are random on the edited rows and +0.0 elsewhere, as
under ``grad_mask``; each arm first takes `--warmup` steps, so the moments are non-zero on the edited rows only (the edit
invariant). Three arms on their own copies of the same tensors: torch.optim.Adam (default: foreach), torch.optim.Adam
(fused=True), MaskedAdam. Each region times `--steps` steps with CUDA events; the arms alternate region by region and
the line reports the median ms per step.
Bytes model (host, from the mask): MaskedAdam touches the mask (P bytes) and, of p, g, m and v, the 32-byte sectors
holding an edited element (read p, g, m, v; write p, m, v: 7 sector transfers each). Fused Adam's model is 7 full
passes over the 59 floats per Gaussian. Achieved bytes/s is model bytes over the median time, against the H100 SXM's
3.35 TB/s of HBM3 (the step is memory-bound: ~10 flops per 28 bytes).
Edit loop: run_edit_loop(grad_mask="kernel") with optimizer="adam" against "masked", eager and with cuda_graph=True,
alternated `--loop-regions` times; median ms/step. The GPU name and power limit (NVML, read only) come from the same run.
One JSON line.
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
from gaussianeditor_b200 import MaskedAdam, synth  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
GROUPS = [("xyz", (3,), 1.6e-5), ("f_dc", (1, 3), 2.5e-3), ("f_rest", (15, 3), 1.25e-4), ("opacity", (1,), 0.1),
          ("scaling", (3,), 1e-2), ("rotation", (4,), 2e-3)]


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


def sectors_touched(mask: np.ndarray, D: int) -> int:
    """32-byte sectors of a row-major float32 [P, D] tensor (32-byte aligned) that hold an element of an edited row."""
    rows = np.nonzero(mask)[0].astype(np.int64)
    first, last = rows * D // 8, (rows * D + D - 1) // 8
    hit = np.zeros((mask.size * D + 7) // 8, dtype=bool)
    for k in range(int((last - first).max(initial=0)) + 1):
        sel = first + k <= last
        hit[(first + k)[sel]] = True
    return int(hit.sum())


def masked_bytes(mask: np.ndarray) -> int:
    return mask.size + sum(7 * 32 * sectors_touched(mask, int(np.prod(shape))) for _, shape, _ in GROUPS)


def optimizer_step(cfg, a, dev):
    cloud, _ = synth.make_config(cfg)
    P = cloud.means3D.shape[0]
    xyz = torch.from_numpy(cloud.means3D).to(dev)
    d = xyz.norm(dim=1)
    masks = {"all": torch.ones(P, dtype=torch.bool, device=dev), "spatial20": d <= torch.quantile(d, 0.2),
             "spatial5": d <= torch.quantile(d, 0.05)}
    gen = torch.Generator(device=dev).manual_seed(0)
    init = [torch.randn((P,) + shape, generator=gen, device=dev) for _, shape, _ in GROUPS]
    out = {"P": P}
    for mname, mask in masks.items():
        grads = [torch.randn((P,) + shape, generator=gen, device=dev) * mask.view((P,) + (1,) * len(shape))
                 for _, shape, _ in GROUPS]
        arms = {}
        for arm in ("adam_foreach", "adam_fused", "masked"):
            params = [torch.nn.Parameter(t.clone()) for t in init]
            for p, g in zip(params, grads):
                p.grad = g
            groups = [{"params": [p], "lr": lr, "name": n} for p, (n, _, lr) in zip(params, GROUPS)]
            if arm == "masked":
                opt = MaskedAdam(groups, eps=1e-15, mask=mask)
            else:
                opt = torch.optim.Adam(groups, eps=1e-15, fused=(arm == "adam_fused"))
            arms[arm] = opt
        for opt in arms.values():
            for _ in range(a.warmup):
                opt.step()
        torch.cuda.synchronize()
        times = {arm: [] for arm in arms}
        for _ in range(a.regions):
            for arm, opt in arms.items():
                def run(opt=opt):
                    for _ in range(a.steps):
                        opt.step()
                times[arm].append(timed(run) / a.steps)
        mnp = mask.cpu().numpy()
        mb, fb = masked_bytes(mnp), 7 * 4 * 59 * P
        res = {"mask_fraction": float(mnp.mean()), "masked_model_bytes": mb, "fused_model_bytes": fb}
        for arm, t in times.items():
            res[arm] = {"ms_per_step": statistics.median(t), "regions": [round(x, 4) for x in t]}
        res["masked"]["achieved_TBps"] = mb / (res["masked"]["ms_per_step"] * 1e-3) / 1e12
        res["masked"]["share_of_3.35TBps"] = mb / (res["masked"]["ms_per_step"] * 1e-3) / HBM_BYTES_PER_S
        res["adam_fused"]["achieved_TBps"] = fb / (res["adam_fused"]["ms_per_step"] * 1e-3) / 1e12
        res["masked_over_foreach"] = res["masked"]["ms_per_step"] / res["adam_foreach"]["ms_per_step"]
        res["masked_over_fused"] = res["masked"]["ms_per_step"] / res["adam_fused"]["ms_per_step"]
        out[mname] = res
        del arms, grads
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--loop-steps", type=int, default=200)
    ap.add_argument("--loop-regions", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda")
    out = {"device": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "steps_per_region": a.steps,
           "regions": a.regions}
    for cfg in ("c3", "c5"):
        out[f"optimizer_{cfg}"] = optimizer_step(cfg, a, dev)

    from gaussianeditor_b200.edit_loop import run_edit_loop
    loop = {}
    for graph in (False, True):
        t = {"adam": [], "masked": []}
        for _ in range(a.loop_regions):
            for arm in t:
                r = run_edit_loop(GaussianRasterizer, steps=a.loop_steps, grad_mask="kernel", optimizer=arm,
                                  cuda_graph=graph)
                t[arm].append(r["ms_per_step"])
        key = "cuda_graph" if graph else "eager"
        loop[key] = {arm: {"ms_per_step": statistics.median(v), "runs": [round(x, 4) for x in v]} for arm, v in t.items()}
        loop[key]["masked_over_adam"] = loop[key]["masked"]["ms_per_step"] / loop[key]["adam"]["ms_per_step"]
    out["c5_edit_loop"] = loop
    print(json.dumps(out))


if __name__ == "__main__":
    main()
