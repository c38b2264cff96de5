"""The rasterizer under the cameras GaussianEditor renders and synth.look_at_camera never builds (synth.camera_family):
unequal focal lengths (PINHOLE intrinsics, the COLMAP reader's resized frames), rolled and arbitrary rotations, fields of
view of 120 and 4 degrees, a camera looking straight down, and a camera inside the cloud.

A look-at camera has square pixels (focal_x and focal_y equal to an ulp) and no roll (view[4] = 0), so a kernel that used
the x focal length or field of view where it needs the y one, or dropped a rotation entry, passed every other test.

CPU: the family reaches its edges; the fp32 and fp64 oracles give the closed-form 2-D covariance, conic, radius and
centre of an axis-aligned Gaussian on the optical axis under unequal focals and a 90-degree roll; fp64 finite
differences of the oracle's gradients; the render entry point and the edit loop's camera keep the two FoVs apart.
GPU, on every camera of the family unless noted:
  * forward, markVisible and apply_weights against the reference's CUDA build, bit for bit;
  * every gradient of the colour, colour + depth and colour + alpha losses (default and deterministic mode) and of the
    fused-activation colour loss against fp64, to max(5e-5, 2 d32), d32 being the distance from fp64 of the fp32 CPU
    oracle (the reference's arithmetic) on the same case and loss;
  * camera-pose gradients against the fp64 autograd truth of test_camera_grad_truth, and the pose chain from a base
    pose equal to the `general` camera;
  * the dense and sparse sharded paths on virtual ranks at world 2 and 3 against the single GPU.
"""
import math
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import synth
from oracle import cpu_oracle as O
from util import cloud_tensors, rel_l2, run_ours, settings_from

CASES = ["aniso_0.5", "aniso_2", "pinhole_resized", "wide_120", "tele_4", "roll_90", "general", "nadir", "inside"]
BG = (0.2, 0.1, 0.3)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "parity", "camera_models_reference.npz")
_FAMILY = {}


def _family():
    if not _FAMILY:
        _FAMILY.update(synth.camera_family())
        assert sorted(_FAMILY) == sorted(CASES)
    return _FAMILY


def _focals(cam):
    """(fx, fy) in pixels as the kernels compute them from the float32 tangents, in fp64."""
    return (cam.image_width / (2.0 * float(np.float32(cam.tanfovx))),
            cam.image_height / (2.0 * float(np.float32(cam.tanfovy))))


def _view_coords(cloud, cam):
    V = cam.viewmatrix.astype(np.float64).T
    return cloud.means3D.astype(np.float64) @ V[:3, :3].T + V[:3, 3]


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_family_reaches_its_edges():
    fam = _family()
    for name, (cloud, cam) in fam.items():
        assert cam.image_width <= 640 and cam.image_width * cam.image_height <= 640 * 480, name
        R = cam.viewmatrix[:3, :3].astype(np.float64)
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-6) and np.linalg.det(R) > 0, name
    ratio = lambda n: _focals(fam[n][1])[1] / _focals(fam[n][1])[0]
    assert abs(ratio("aniso_0.5") - 0.5) < 1e-6 and abs(ratio("aniso_2") - 2.0) < 1e-6
    assert abs(ratio("pinhole_resized") - 1090.0 / 1160.0) < 1e-6
    assert abs(_focals(fam["pinhole_resized"][1])[0] - 1160.0 * 512 / 840) < 1e-3   # the 840-px side scaled to 512
    assert abs(fam["wide_120"][1].tanfovx - math.tan(math.radians(60))) < 1e-9 and fam["wide_120"][1].tanfovy > 1.0
    assert abs(fam["tele_4"][1].tanfovx - math.tan(math.radians(2))) < 1e-9 and _focals(fam["tele_4"][1])[0] > 9000
    # every entry of the view rotation reaches 0.3 in magnitude on some camera
    views = np.stack([c.viewmatrix[:3, :3] for _, c in fam.values()])
    assert (np.abs(views) >= 0.3).any(0).all(), np.abs(views).max(0)
    roll = fam["roll_90"][1].viewmatrix.reshape(-1)
    assert roll[0] == 0.0 and abs(roll[4]) == 1.0
    assert abs(fam["nadir"][1].viewmatrix.reshape(-1)[6]) == 1.0          # camera z = world y
    assert np.abs(fam["general"][1].viewmatrix[:3, :3]).min() >= 0.05
    for name, (cloud, cam) in fam.items():
        f = O.forward_from(cloud, cam, f32=False, render=False)
        vis = f.radii > 0
        pv = _view_coords(cloud, cam)
        clamped = (np.abs(pv[:, 0] / pv[:, 2]) > 1.3 * np.float32(cam.tanfovx)) | \
                  (np.abs(pv[:, 1] / pv[:, 2]) > 1.3 * np.float32(cam.tanfovy))
        band = (pv[:, 2] > 0.2) & (pv[:, 2] < 0.3) & vis
        covers = f.tiles_touched == f.ranges.shape[0]
        f.close()
        assert vis.sum() >= 200, name
        if name in ("wide_120", "tele_4"):
            assert (clamped & vis).sum() >= 100, (name, (clamped & vis).sum())
        if name == "inside":
            assert (pv[:, 2] < 0).sum() >= 1000 and band.sum() >= 20 and covers.sum() >= 1, \
                ((pv[:, 2] < 0).sum(), band.sum(), covers.sum())


def _on_axis(R, W=640, H=480, fx=520.0, fy=260.0, z=3.0, abc=(0.05, 0.012, 0.07)):
    """One axis-aligned Gaussian with scales abc on the optical axis at depth z -> (Cloud, Camera)."""
    cam = synth.pinhole_camera(R, np.zeros(3), W, H, fx, fy)
    xyz = (np.asarray(R, np.float64).T @ np.array([0.0, 0.0, z]))[None]
    cloud = synth.Cloud(xyz.astype(np.float32), np.array([abc], np.float32), np.array([[1, 0, 0, 0]], np.float32),
                        np.array([[0.7]], np.float32), np.zeros((1, 1, 3), np.float32), 0)
    return cloud, cam


@pytest.mark.parametrize("f32", [False, True], ids=["fp64", "fp32"])
@pytest.mark.parametrize("roll", [False, True], ids=["world_axes", "roll_90"])
def test_closed_form_on_axis(roll, f32):
    """cov2D = diag((fx a / z)^2, (fy b / z)^2) + 0.3 for a camera whose axes are the world's, and diag((fx b / z)^2,
    (fy a / z)^2) + 0.3 under the 90-degree roll (camera x = world y); the conic is its inverse, the radius
    ceil(3 sqrt(lambda_max)) (the reference's 0.1 floor under the eigenvalue spread), the centre the frame's centre."""
    R = np.array([[0.0, 1, 0], [-1, 0, 0], [0, 0, 1]]) if roll else np.eye(3)
    z, (a, b, c) = 3.0, (0.05, 0.012, 0.07)
    cloud, cam = _on_axis(R, z=z, abc=(a, b, c))
    fx, fy = _focals(cam)
    sx, sy = (b, a) if roll else (a, b)
    sx, sy = float(np.float32(sx)), float(np.float32(sy))
    dil = float(np.float32(0.3))                   # the low-pass 0.3f of the kernels and both oracles
    va, vc = (fx * sx / z) ** 2 + dil, (fy * sy / z) ** 2 + dil
    assert abs(va - vc) > 10.0                     # the two axes are told apart
    mid = 0.5 * (va + vc)
    lam = mid + math.sqrt(max(0.1, mid * mid - va * vc))
    r = 3.0 * math.sqrt(lam)
    assert 0.05 < r - math.floor(r) < 0.95         # the radius is not at a rounding edge
    f = O.forward_from(cloud, cam, f32=f32)
    tol = 2e-6 if f32 else 1e-10
    co = f.conic_opacity[0].astype(np.float64)
    assert abs(co[0] * va - 1) <= tol and abs(co[2] * vc - 1) <= tol and abs(co[1]) <= tol * abs(co[0]), (co, va, vc)
    assert f.radii[0] == math.ceil(r), (f.radii[0], r)
    W, H = cam.image_width, cam.image_height
    assert np.allclose(f.means2D[0], [(W - 1) / 2, (H - 1) / 2], rtol=0, atol=1e-4 if f32 else 1e-9)
    assert abs(f.depths[0] - z) <= (1e-6 if f32 else 1e-12)
    f.close()


@pytest.mark.parametrize("case", ["aniso_2", "general", "wide_120"])
def test_gradients_match_fp64_finite_differences(case):
    """test_oracle_kat's directional finite differences on the case's camera, with 24 Gaussians in its view space (none
    at the Jacobian clamp, whose gradient convention is not the derivative of the clamped map), at depths beyond 4.
    Their sizes are set to 1..3 px per axis: the check skips every direction in which some pixel's alpha crosses
    1/255, and the contours of larger splats on a frame this size are long enough that almost every direction crosses
    one."""
    from test_oracle_kat import check_finite_differences
    cam = _family()[case][1]
    cloud = synth.view_space_cloud(cam, 400, seed=7, near_frac=0.0, clamp_frac=0.0, beyond_frac=0.0)
    z = _view_coords(cloud, cam)[:, 2]
    keep = np.flatnonzero(z > 4.0)[:24]        # world-sized scales: the fixed finite-difference steps stay small
    cloud = synth.Cloud(*(np.ascontiguousarray(getattr(cloud, k)[keep]) for k in
                          ("means3D", "scales", "rotations", "opacities", "shs")), 3)
    rng = np.random.default_rng(43)
    cloud.scales = (z[keep, None] * rng.uniform(1.0, 3.0, (24, 3)) / max(_focals(cam))).astype(np.float32)
    G = rng.uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32).astype(np.float64)
    g = check_finite_differences(cloud, cam, G, BG, rng)
    assert (np.abs(g["dmean3D"]).sum(1) > 0).sum() >= 12


def _editor_camera():
    """GaussianEditor's camera for the pinhole_resized case: FoVx and FoVy from different focal lengths."""
    from gaussianeditor_b200 import edit_loop
    cam = _family()["pinhole_resized"][1]
    return cam, edit_loop.make_view(cam, "cpu")


def test_render_and_edit_loop_keep_both_fovs():
    """The render entry point passes tan(FoVx / 2) and tan(FoVy / 2) separately, and the edit loop's camera conversion
    round-trips a camera whose FoVs come from different focal lengths."""
    from gaussianeditor_b200 import gaussian_renderer
    cam, view = _editor_camera()
    assert abs(view.FoVx - 2 * math.atan(cam.image_width / (2 * 1160.0 * 512 / 840))) < 1e-12
    rs = gaussian_renderer._settings_for(view, torch.zeros(3), 1.0, 3)
    assert rs.tanfovx == math.tan(0.5 * view.FoVx) and rs.tanfovy == math.tan(0.5 * view.FoVy)
    assert abs(rs.tanfovx / cam.tanfovx - 1) < 1e-12 and abs(rs.tanfovy / cam.tanfovy - 1) < 1e-12
    assert abs((rs.tanfovx / rs.tanfovy) / (cam.image_width / cam.image_height) - 1) > 0.05   # not square pixels
    assert (rs.image_width, rs.image_height) == (cam.image_width, cam.image_height)
    assert np.array_equal(rs.viewmatrix.numpy(), cam.viewmatrix) and np.array_equal(rs.projmatrix.numpy(), cam.projmatrix)
    assert np.array_equal(rs.campos.numpy(), cam.campos)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _masks(cam):
    rng = np.random.default_rng(19)
    H, W = cam.image_height, cam.image_width
    return (rng.uniform(size=(1, H, W)) > 0.5).astype(np.float32), rng.uniform(size=(3, H, W)).astype(np.float32)


def _apply_weights(rast_or_ref, ct, P, mask, rs=None):
    w = torch.zeros(P, mask.shape[0], device="cuda")
    c = torch.zeros(P, 1, dtype=torch.int32, device="cuda")
    m = torch.from_numpy(mask).cuda()
    if rs is None:
        rast_or_ref.apply_weights(ct["means3D"], None, ct["opacities"], None, w, ct["scales"], ct["rotations"], None, c, m)
    else:
        rast_or_ref.apply_weights(means3D=ct["means3D"], opacities=ct["opacities"], scales=ct["scales"],
                                  rotations=ct["rotations"], weights=w, cnt=c, image_weights=m, bg=rs.bg,
                                  viewmatrix=rs.viewmatrix, projmatrix=rs.projmatrix, campos=rs.campos,
                                  tanfovx=rs.tanfovx, tanfovy=rs.tanfovy, image_height=mask.shape[1],
                                  image_width=mask.shape[2])
    torch.cuda.synchronize()
    return w, c


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_forward_mark_visible_apply_weights_match_reference(case):
    """Every forward output (radii, tile lists, n_contrib, final_T and so alpha, colour, depth, the per-Gaussian
    records) bit for bit the reference's; markVisible bit for bit; apply_weights with a binary single-channel mask
    bit for bit and with a float three-channel mask to summation order (the reference adds with float atomics)."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    from oracle import ref_cuda
    from test_parity_gpu import _Ref, _digest, _ours_forward_fields, _ref_forward_fields, _ref_run
    cloud, cam = _family()[case]
    P = cloud.means3D.shape[0]
    ours = _ours_forward_fields(run_ours(cloud, cam, BG))
    ct = cloud_tensors(cloud, "cuda")
    rs = settings_from(cam, BG, cloud.sh_degree, "cuda")
    rast = GaussianRasterizer(rs)
    vis = rast.markVisible(ct["means3D"])
    binary, soft = _masks(cam)
    wb, cb = _apply_weights(rast, ct, P, binary)
    ws, cs = _apply_weights(rast, ct, P, soft)

    def compute():
        out = {f"fwd/{k}": x for k, x in _ref_forward_fields(_ref_run(cloud, cam, BG)).items()}
        R = ref_cuda.ReferenceRasterizer()
        out["visible"] = R.mark_visible(ct["means3D"], rs.viewmatrix, rs.projmatrix)
        out["binary/weights"], out["binary/cnt"] = _apply_weights(R, ct, P, binary, rs)
        out["soft/weights"], out["soft/cnt"] = _apply_weights(R, ct, P, soft, rs)
        return out
    ref = _Ref(f"camera_models/{case}", compute, close=("soft/weights",), golden=GOLDEN)
    bad = [k for k, x in ours.items() if not ref.equal(f"fwd/{k}", x)]
    assert not bad, (case, bad)
    assert ours["R"] > 0 and int(cb.sum()) > 0
    assert ref.equal("visible", vis)
    assert ref.equal("binary/cnt", cb) and ref.equal("binary/weights", wb)
    assert ref.equal("soft/cnt", cs)
    g, r = ref.pair("soft/weights", ws)
    assert rel_l2(g, r) <= 1e-5 and np.abs(g - r).max() <= 1e-4 * ref.absmax("soft/weights")
    assert _digest(cs) == _digest(cb * 3)      # cnt advances by CH per hit


_MATCHED = {}


def _matched_case(case):
    """The case's cloud without the rows whose radii differ between the GPU and the fp64 oracle (a radius step or the
    near cut decided the other way by rounding), so that both sides sum over the same splats."""
    from test_camera_grad_truth import _matched
    if case not in _MATCHED:
        cloud, cam = _family()[case]
        _MATCHED.clear()
        _MATCHED[case] = (_matched(cloud, cam)[0], cam)
    return _MATCHED[case]


def _upstreams(cam, seed):
    from test_deterministic_truth import _upstreams as up
    return up(cam, seed)


def _check(got, truth, truth32, label, skip=()):
    """rel. L2 of every gradient from fp64 <= max(5e-5, 2 d32), d32 the fp32 oracle's own distance from fp64."""
    from test_deterministic_truth import _truth_errors
    errs = _truth_errors(got, truth, skip)
    d32 = _truth_errors({k: np.asarray(truth32[k]).reshape(np.shape(got[k])) for k in errs}, truth, skip)
    bound = {k: max(5e-5, 2.0 * d32[k]) for k in errs}
    print(label, {k: f"{errs[k]:.2e} (fp32 {d32[k]:.2e})" for k in errs})
    bad = {k: (errs[k], bound[k]) for k in errs if not errs[k] <= bound[k]}
    assert not bad, (label, bad)


# On aniso_2 the reference's own CUDA build misses fp64 as far as ours: measured on an H100 (colour loss), dmean3D
# 1.02e-4 from fp64 for both, 2.4e-6 between them, while the fp32 CPU oracle is 7.2e-6 away; 99.8 % of the squared
# error sits on five Gaussians. The GPU arithmetic both builds share (FMA contraction), not the port, decides it.
_SHARED_WITH_REFERENCE = pytest.mark.xfail(strict=True, reason="the reference CUDA build misses fp64 by the same 1e-4")
BACKWARD_CASES = [pytest.param(c, marks=_SHARED_WITH_REFERENCE) if c == "aniso_2" else c for c in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize("deterministic", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("form", ["colour", "depth", "alpha"])
@pytest.mark.parametrize("case", BACKWARD_CASES)
def test_backward_against_fp64(case, form, deterministic):
    from test_deterministic_truth import _run, _truth
    cloud, cam = _matched_case(case)
    gC, gD = _upstreams(cam, 71)
    got, _ = _run(cloud, cam, BG, gC, gD=gD if form == "depth" else None, gA=gC[0] if form == "alpha" else None,
                  deterministic=deterministic)
    truth = _truth(cloud, cam, BG, form, gC, gD)
    truth32 = _truth(cloud, cam, BG, form, gC, gD, f32=True)
    _check(got, truth, truth32, (case, form, deterministic))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_fused_activation_backward_against_fp64(case):
    """forward_raw (deterministic) on the case's cloud in raw form: every raw gradient against the fp64 chain of the
    fp64 oracle, to max(5e-5, 2 d32) with d32 from the fp32 oracle's gradients chained in fp64."""
    from test_fused_activation_truth import KEYS, chain, cloud_of, raw_truth, run_fused, to_raw
    cloud, cam = _matched_case(case)
    raw = to_raw(cloud, seed=3)
    gC, _ = _upstreams(cam, 73)
    out, got = run_fused(raw, cloud.sh_degree, cam, BG, gC=gC, deterministic=True)
    truth, radii = raw_truth(raw, cloud.sh_degree, cam, BG, gC=gC)
    f = O.forward_from(cloud_of(raw, cloud.sh_degree), cam, BG, f32=True)
    truth32 = chain(raw, f.backward(gC))
    f.close()
    assert np.array_equal(out[1], radii)
    _check({k: got[k] for k in KEYS}, truth, truth32, (case, "raw"))


CAMERA_CASES = ["aniso_2", "roll_90", "general", "wide_120", "inside"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CAMERA_CASES)
def test_camera_gradients_against_fp64(case):
    """The camera-pose gradients (colour + depth loss) against test_camera_grad_truth's fp64 autograd truth, element
    by element (TAU) and per array (RHO), and the world-translation identity."""
    from test_camera_grad_truth import _compare
    cloud, cam = _family()[case]
    _compare(cloud, cam, case, depth=True, seed=8)


@pytest.mark.gpu
def test_pose_chain_from_the_general_camera():
    """pose.grad from a base pose equal to the `general` camera (a rotation with every entry at least 0.05), not a
    small nudge of a look-at camera: the pose is that rotation as an axis-angle and its translation, applied to the
    identity."""
    from scipy.spatial.transform import Rotation
    from test_camera_grad_truth import pose_chain
    cloud, cam = _family()["general"]
    W2C = cam.viewmatrix.astype(np.float64).T
    p0 = np.concatenate([Rotation.from_matrix(W2C[:3, :3]).as_rotvec(), W2C[:3, 3]])
    assert np.linalg.norm(p0[:3]) > 1.0
    pose_chain(cloud, cam, np.eye(4), p0, "pose_chain/general")


SHARD_CASES = ["aniso_2", "general", "inside"]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("case", SHARD_CASES)
def test_sharded_paths_match_single_gpu(case, world):
    """Dense and sparse virtual ranks (test_sharded's harness): frames, depth, radii and the instance total bit for bit
    the single GPU's, default gradients to summation order; the deterministic backward: dense and sparse equal bit for
    bit, and both equal the single GPU's deterministic backward to summation order (test_sharded_deterministic)."""
    from test_sharded import virtual_dense, virtual_sparse
    from test_sharded_deterministic import _dense_grads, _equal, _inputs, _single_grads, _sparse_grads
    cloud, cam = _family()[case]
    gC, _ = _upstreams(cam, 75)
    sc = dict(cloud=cloud, cam=cam, bg=BG, dL=gC, ref=run_ours(cloud, cam, bg=BG, dL=gC))
    virtual_dense(sc, world)
    virtual_sparse(sc, world, "tight", max_fill=1.0)   # 13 tile rows on aniso_2: many splats reach both ranks
    rs = settings_from(cam, BG, cloud.sh_degree, "cuda")
    d = _inputs(cloud_tensors(cloud, "cuda"), colors=False, cov=False)
    dL = torch.from_numpy(gC).cuda()
    single = _single_grads(rs, d, dL)
    dense = _dense_grads(world, rs, d, dL)
    _equal(dense, _sparse_grads(world, rs, d, dL, "tight"))
    assert dense.keys() == single.keys()
    for k in single:
        assert rel_l2(dense[k].cpu().numpy(), single[k].cpu().numpy()) <= 2e-5, (case, world, k)


@pytest.mark.gpu
def test_render_passes_both_fovs():
    """gaussian_renderer.render on GaussianEditor's camera with FoVx and FoVy from different focal lengths draws the
    same image, bit for bit, as the rasterizer built from the camera's own tangents."""
    from gaussianeditor_b200 import edit_loop, gaussian_renderer
    cloud, cam = _family()["pinhole_resized"]
    view = edit_loop.make_view(cam, "cuda")
    ct = cloud_tensors(cloud, "cuda")
    pc = SimpleNamespace(get_xyz=ct["means3D"], get_opacity=ct["opacities"], get_scaling=ct["scales"],
                         get_rotation=ct["rotations"], get_features=ct["shs"], active_sh_degree=cloud.sh_degree)
    got = gaussian_renderer.render(view, pc, SimpleNamespace(), torch.tensor(BG, dtype=torch.float32, device="cuda"))
    want = run_ours(cloud, cam, BG)
    assert torch.equal(got["radii"], want["radii"]) and torch.equal(got["render"].detach(), want["color"])
