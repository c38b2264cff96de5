"""Golden vectors produced by the REFERENCE's own CUDA build (oracle/_ref, i.e. the unmodified reference .cu files)
with tools/make_golden.py and committed under tests/golden/ (forward outputs are the same on every GPU the reference
was run on; gradients differ only by the order of its float atomics).

  * CPU (no GPU needed): the oracle restatement reproduces them -- integers exactly (up to the documented FMA-contraction
    slack), floats to tolerance. This is what pins the oracle to the real reference when no GPU is at hand.
  * GPU: our kernels reproduce the forward outputs BIT-FOR-BIT and the gradients to tolerance.
"""
import glob
import os

import numpy as np
import pytest

from gaussianeditor_b200 import synth
from oracle import cpu_oracle as O

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "*.npz")))
GRAD_KEYS = [("dmean3D", "dL_dmeans3D"), ("dmean2D", "dL_dmeans2D"), ("dopacity", "dL_dopacity"),
             ("dscale", "dL_dscales"), ("drot", "dL_drotations"), ("dsh", "dL_dsh"), ("dcolor", "dL_dcolors")]


def _load(path):
    z = np.load(path)
    cloud = synth.Cloud(z["means3D"], z["scales"], z["rotations"], z["opacities"], z["shs"], int(z["sh_degree"]))
    cam = synth.Camera(int(z["H"]), int(z["W"]), float(z["tanfovx"]), float(z["tanfovy"]), z["viewmatrix"],
                       z["projmatrix"], z["campos"])
    cp = z["colors_precomp"] if z["colors_precomp"].size else None
    return z, cloud, cam, cp


def test_golden_files_present():
    assert len(GOLDEN) >= 3, "tests/golden/*.npz missing (generate with tools/make_golden.py on a GPU box)"


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_cpu_oracle_reproduces_reference_golden(path):
    z, cloud, cam, cp = _load(path)
    f = O.forward_from(cloud, cam, bg=z["bg"], colors_precomp=cp, scale_modifier=float(z["scale_modifier"]))
    assert np.array_equal(f.radii, z["radii"])
    tiles_equal = np.array_equal(f.tiles_touched, z["tiles_touched"].astype(np.uint32))
    assert (f.tiles_touched != z["tiles_touched"].astype(np.uint32)).sum() <= 1
    if tiles_equal:
        assert f.num_rendered == int(z["R"])
        assert np.array_equal(f.ranges, z["ranges"].astype(np.uint32))
        assert np.array_equal(f.point_list, z["point_list"].astype(np.uint32))
        assert (f.n_contrib != z["n_contrib"].astype(np.uint32)).mean() <= 1e-3
    vis = z["radii"] > 0
    assert np.allclose(f.means2D[vis], z["means2D"][vis], rtol=1e-5, atol=1e-4)
    assert np.allclose(f.depths[vis], z["depths"][vis], rtol=1e-6)
    if cp is None:
        assert np.allclose(f.rgb[vis], z["rgb"][vis], atol=2e-6)
    bad = np.abs(f.color - z["color"]) > 1e-5 + 1e-4 * np.abs(z["color"])
    assert bad.mean() <= 2e-3, bad.mean()
    assert np.allclose(f.final_T, z["final_T"], atol=2e-5)
    g = f.backward(z["dL"])
    for a, b in GRAD_KEYS:
        if a == "dsh" and cp is not None:
            continue
        ref = z[b]
        err = np.linalg.norm(g[a].reshape(ref.shape) - ref) / max(np.linalg.norm(ref), 1e-30)
        assert err <= 2e-4, (a, err)
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_gpu_kernels_reproduce_reference_golden(path):
    from util import run_ours
    z, cloud, cam, cp = _load(path)
    out = run_ours(cloud, cam, tuple(z["bg"]), dL=z["dL"], colors_precomp=cp, scale_modifier=float(z["scale_modifier"]))
    v = out["views"]
    assert out["R"] == int(z["R"])
    assert np.array_equal(out["radii"].cpu().numpy(), z["radii"])
    assert np.array_equal(v["ranges"].cpu().numpy(), z["ranges"])
    assert np.array_equal(v["point_list"].cpu().numpy(), z["point_list"])
    assert np.array_equal(v["n_contrib"].cpu().numpy(), z["n_contrib"])
    assert np.array_equal(v["final_T"].cpu().numpy(), z["final_T"])          # bit-exact
    assert np.array_equal(out["color"].cpu().numpy(), z["color"])            # bit-exact
    assert np.array_equal(out["depth"].cpu().numpy(), z["depth"])            # bit-exact
    noise = dict(zip([str(k) for k in z["noise_keys"]], z["noise"]))
    for a, b in GRAD_KEYS:
        g = out["grads"][a]
        if g is None:
            continue
        ref = z[b]
        err = np.linalg.norm(g.cpu().numpy().reshape(ref.shape) - ref) / max(np.linalg.norm(ref), 1e-30)
        assert err <= 1e-4 + 10 * noise.get(b, 0.0), (a, err)
