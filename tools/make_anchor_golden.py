"""Record what GaussianEditor's own ``GaussianModel.anchor_loss`` computes, for tests/test_anchor_loss.py:

    python tools/make_anchor_golden.py <GaussianEditor checkout> tests/golden/anchor/reference_anchor.npz

The reference's ``scene/gaussian_model.py`` is imported unchanged on the CPU, with the third-party modules absent
here stubbed (``install_stubs`` of make_caller_golden.py). Each model is made with ``GaussianModel.__new__`` plus
attributes, so nothing touches a CUDA device. Per case the file holds the inputs (six parameters, their anchors, the
mask, the generations, the weight schedule), the four returned values in the reference dict's order, and the six
parameter gradients after ``sum(lambda * value).backward()``. Cases: SH degree 3 and 0, P in {1, 33, 257}, random /
all / empty masks, and a three-generation schedule whose youngest generation has weight 0."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_caller_golden import install_stubs   # noqa: E402

TERMS = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")
# GaussianEditor's configs/edit-*.yaml weights (color, geo, opacity, scale): the color term gets a gradient too
LAMBDA = {"loss_anchor_color": 5.0, "loss_anchor_geo": 50.0, "loss_anchor_opacity": 50.0, "loss_anchor_scale": 50.0}
SCHEDULE = np.array([0.0169, 0.01, 0.0], dtype=np.float32)   # after two densifications: g0, g1, newborn g2


def shapes(P, deg):
    return {"_xyz": (P, 3), "_features_dc": (P, 1, 3), "_features_rest": (P, (deg + 1) ** 2 - 1, 3),
            "_scaling": (P, 3), "_rotation": (P, 4), "_opacity": (P, 1)}


def make_case(P, deg, mask_kind, seed):
    rng = np.random.default_rng(seed)
    params, anchors = {}, {}
    for k, s in shapes(P, deg).items():
        a = rng.standard_normal(s).astype(np.float32)
        params[k] = (a + 0.1 * rng.standard_normal(s)).astype(np.float32)
        anchors[k] = a
    mask = {"random": rng.random(P) < 0.4, "all": np.ones(P, bool), "empty": np.zeros(P, bool)}[mask_kind]
    if mask_kind == "random" and P > 1:
        mask[0] = True   # at least one edited row
    generation = rng.integers(0, len(SCHEDULE), P).astype(np.int64)
    return params, anchors, mask, generation


def main(ref_root, out):
    sys.path.insert(0, ref_root)
    install_stubs()
    import gaussiansplatting.scene.gaussian_model as GM
    rec, cases = {}, []
    seed = 0
    for deg in (3, 0):
        for P in (1, 33, 257):
            for mask_kind in ("random", "all", "empty"):
                name = f"d{deg}_p{P}_{mask_kind}"
                params, anchors, mask, generation = make_case(P, deg, mask_kind, seed)
                seed += 1
                m = GM.GaussianModel.__new__(GM.GaussianModel)
                for k in TERMS:
                    setattr(m, k, torch.from_numpy(params[k].copy()).requires_grad_(True))
                m.anchor = {k: torch.from_numpy(anchors[k].copy()) for k in TERMS}
                m.mask = torch.from_numpy(mask.copy())
                m._generation = torch.from_numpy(generation.copy())
                m._anchor_loss_schedule = torch.from_numpy(SCHEDULE.copy())
                res = m.anchor_loss()
                keys = list(res)
                loss = 0
                for k, v in res.items():
                    loss = loss + v * LAMBDA[k]
                loss.backward()
                for k in TERMS:
                    rec[f"{name}/param/{k}"] = params[k]
                    rec[f"{name}/anchor/{k}"] = anchors[k]
                    rec[f"{name}/grad/{k}"] = getattr(m, k).grad.numpy()
                rec[f"{name}/mask"] = mask
                rec[f"{name}/generation"] = generation
                rec[f"{name}/schedule"] = SCHEDULE
                rec[f"{name}/out"] = np.array([float(res[k].detach()) for k in keys], dtype=np.float32)
                cases.append(name)
    meta = {"cases": cases, "keys": keys, "lambda": LAMBDA, "terms": list(TERMS)}
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, meta=np.array(json.dumps(meta, sort_keys=True)), **rec)
    print("wrote", out, len(cases), "cases")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
