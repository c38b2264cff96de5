"""The rasterizer at the magnitudes trained clouds reach (synth.magnitude_cloud, synth.rescaled_patch): scales that vanish
or overflow in fp32, screen radii at and past 2^24 and 2^31, 2-D covariances whose determinant rounding decides, and
scenes translated far from the origin or rescaled together with their camera.

There the result is decided by conversion and NaN rules, not by ordinary arithmetic: float -> int of the radius and of
the tile rectangle saturates on the GPU (cvt.rzi.s32.f32: NaN -> 0, out of range -> INT_MIN / INT_MAX) where a host
(int) cast gives INT_MIN; fminf(0.99, o exp(NaN)) = 0.99 blends a NaN-conic splat at 0.99 over its rectangle; the hit
test !(power > 0) lets a NaN power through. Every input is finite; only intermediates overflow.

CPU: the generator is seeded and every group reaches its edge (synth.preprocess_fp32, the kernels' arithmetic, and the
fp64 oracle); the oracle's known answers (radius INT_MAX over the whole grid for a 1e18 Gaussian in both modes, radius
3 for a vanishing one); rectangles inside the grid and R far below any capacity before anything is launched; the
sub-block culling predicate misses no (pixel, splat) pair of the scene.
GPU, with the shipped options unless noted:
  * every forward output bit for bit the reference's CUDA build (or the digests recorded from it in
    tests/golden/parity/magnitudes_reference.npz) under every render_fwd variant and both binning and depth-sort
    variants, and our radii the kernels' arithmetic restated in synth.preprocess_fp32;
  * the colour backward, default and deterministic, against the reference: non-finite entries at the same positions,
    finite ones to test_parity_gpu._grads_vs_reference_and_truth's bound; deterministic mode gives the same bits twice;
  * the colour, colour + depth and colour + alpha losses against fp64 on the groups whose intermediates stay finite;
  * the rescaled patches against fp64 within twice the unscaled patch's error + 1e-6, the translated ones bit for bit
    the reference;
  * markVisible and apply_weights (masks in multiples of 2^-8) bit for bit, static capacity at R, grad_mask, and the
    dense and sparse sharded paths on two virtual ranks.
"""
import os

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import synth
from oracle import cpu_oracle as O
from util import cloud_tensors, rel_l2, run_ours, settings_from

BG = (0.2, 0.3, 0.1)
INT_MAX = 2 ** 31 - 1
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "parity", "magnitudes_reference.npz")
# groups whose intermediates stay finite and whose radii the fp32 kernels and fp64 share
FINITE_GROUPS = ("opacity_denormal", "opacity_denormal_min", "opacity_zero", "opacity_255_below", "opacity_255",
                 "opacity_255_above", "opacity_one", "clamp_zero", "vanishing", "vanishing_mixed", "sh_1e30")
SCALES = (1e-2, 1e2, 1e4)
SHIFTS = (1e2, 1e4, 1e5)
_SCENE = {}


def _scene():
    if not _SCENE:
        _SCENE["s"] = synth.magnitude_cloud()
    return _SCENE["s"]


def _sub(cloud, rows):
    return synth.Cloud(*(np.ascontiguousarray(getattr(cloud, k)[rows]) for k in
                         ("means3D", "scales", "rotations", "opacities", "shs")), cloud.sh_degree)


def _finite_scene():
    cloud, cam, groups = _scene()
    return _sub(cloud, np.sort(np.concatenate([groups[g] for g in FINITE_GROUPS]))), cam


def _grid(cam):
    return (cam.image_width + 15) // 16, (cam.image_height + 15) // 16


def _rects(means2D, radii, gx, gy):
    """tile_rect of every splat with the device's saturating conversions (fp32 as the kernels)."""
    px, py = means2D[:, 0].astype(np.float32), means2D[:, 1].astype(np.float32)
    r = radii.astype(np.float32)
    t, one = np.float32(16), np.float32(1)

    def conv(v, n):
        v = np.nan_to_num(v.astype(np.float64), nan=0.0, posinf=2.0 ** 31, neginf=-2.0 ** 31)
        return np.clip(np.trunc(v), 0, n).astype(np.int64)
    with np.errstate(all="ignore"):
        return (conv((px - r) / t, gx), conv((py - r) / t, gy), conv((((px + r) + t) - one) / t, gx),
                conv((((py + r) + t) - one) / t, gy))


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_generator_is_seeded_and_every_group_reaches_its_edge():
    cloud, cam, groups = _scene()
    again = synth.magnitude_cloud()
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        assert np.array_equal(getattr(cloud, k), getattr(again[0], k)), k
    assert {k: v.tolist() for k, v in groups.items()} == {k: v.tolist() for k, v in again[2].items()}
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        assert np.isfinite(getattr(cloud, k)).all(), k                      # only intermediates overflow
    assert cam.image_height % 16 != 0 and cloud.sh_degree == 3
    f = synth.preprocess_fp32(cloud, cam)
    f64 = O.forward_from(cloud, cam, f32=False, render=False)
    try:
        r64, conic64 = f64.radii.astype(np.int64), f64.conic_opacity
        rad, radf, cov2, det, conic = f["radius"], f["radius_f"], f["cov2"], f["det"], f["conic"]
        # vanishing: cov3D denormal or 0 from 1e-19 down, the 2-D covariance the dilation alone, radius 3
        v = groups["vanishing"]
        k = np.round(np.log10(cloud.scales[v, 0].astype(np.float64))).astype(int)
        assert k.tolist() == list(range(-30, -3))
        tiny = np.abs(f["cov3D"][v[k <= -19]])
        assert (tiny < np.finfo(np.float32).tiny).all() and (tiny == 0).any() and (tiny > 0).any()
        exact = v[k <= -10]
        assert (cov2[exact, 0] == np.float32(0.3)).all() and (cov2[exact, 2] == np.float32(0.3)).all()
        assert (np.abs(cov2[exact, 1]) < 1e-17).all() and (det[exact] == np.float32(0.3) * np.float32(0.3)).all()
        assert (rad[v] == 3).all() and (r64[v] == 3).all()          # mid 0.3, det 0.09, disc sqrt(0.1)
        assert (rad[groups["vanishing_mixed"]] > 3).all()
        # radius edges: 3 sqrt(lambda_max) in fp32 just below, on and above 2^24 and 2^31 - 1, and beyond
        e = groups["radius_edge"]
        assert radf[e[:6]].tolist() == list(synth.MAGNITUDE_RADII[:6])
        assert rad[e].tolist() == [16777215, 16777216, 16777218, 2147483520] + [INT_MAX] * 4
        assert (np.abs(r64[e[:3]] - 2 ** 24) < 64).all() and (r64[e[4:]] == INT_MAX).all()
        # overflow: radius INT_MAX in fp32 and fp64; cov2 reaches inf; det -inf or NaN; the conic 0 or NaN
        ov, rot = groups["overflow"], groups["overflow_rotated"]
        assert (rad[ov] == INT_MAX).all() and (rad[rot] == INT_MAX).all() and (r64[ov] == INT_MAX).all()
        assert (r64[rot] == INT_MAX).all()
        assert np.isinf(cov2[ov]).any(1).sum() >= 2 and np.isinf(cov2[rot]).any(1).all()
        assert (np.isinf(det[ov]) | np.isnan(det[ov])).all() and (np.isinf(det[rot]) | np.isnan(det[rot])).all()
        assert np.isnan(conic[rot]).any(1).sum() >= 6 and ((conic[ov] == 0) | np.isnan(conic[ov])).all()
        assert np.isnan(conic[ov]).any(1).sum() >= 2 and (conic[ov] == 0).all(1).sum() >= 5
        assert np.isinf(cov2[rot, 1]).sum() >= 4 and np.isnan(cov2[rot, 1]).sum() >= 2      # b = +-inf and NaN
        assert np.isfinite(f64.cov3D[np.concatenate([ov, rot])]).all() and np.isfinite(conic64[ov]).all()
        # cancelling determinant: exactly 0 (culled), a few ulp above 0 (huge conic), below 0; fp64 keeps det > 0
        cz, ct, cn = groups["cancel_zero"], groups["cancel_tiny"], groups["cancel_negative"]
        assert (det[cz] == 0).all() and (rad[cz] == 0).all() and (cov2[cz] == np.float32(2 ** 24)).all()
        assert (det[ct] > 0).all() and (np.abs(conic[ct]).max(1) >= 1e3).all() and (rad[ct] > 0).all()
        assert (det[cn] < 0).all() and (rad[cn] > 0).all()
        ratio = cloud.scales[np.concatenate([ct, cn])].max(1) / cloud.scales[np.concatenate([ct, cn])].min(1)
        assert ratio.min() >= 1e4 * 0.5 and ratio.max() <= 2e8
        assert (r64[np.concatenate([cz, ct, cn])] > 0).all() and (np.abs(conic64[ct, :3]).max(1) < 10).all()
        # colour and opacity extremes
        o = lambda g: cloud.opacities[groups[g], 0]
        o255 = np.float32(1 / 255)
        assert (o("opacity_zero") == 0).all() and (o("opacity_one") == 1).all() and (o("opacity_255") == o255).all()
        assert (o("opacity_255_below") == np.nextafter(o255, np.float32(0))).all()
        assert (o("opacity_255_above") == np.nextafter(o255, np.float32(1))).all()
        den = np.concatenate([o("opacity_denormal"), o("opacity_denormal_min")])
        assert ((den > 0) & (den < np.finfo(np.float32).tiny)).all()
        assert np.abs(cloud.shs[groups["sh_1e30"]]).max() >= np.float32(1e30)
        # the kernels' colour of clamp_zero: fp32(SH_C0) sh0 + 0.5 = +0 exactly (the other 15 coefficients are 0)
        cz3 = groups["clamp_zero"]
        assert (np.float32(synth.SH_C0) * cloud.shs[cz3, 0, :] + np.float32(0.5) == 0).all()
        assert (cloud.shs[cz3, 1:, :] == 0).all()
        # no visible row with a NaN radius (it would convert to 0 and leave the reference's instance slots unwritten)
        live = (f["depth"] > np.float32(0.2)) & (det != 0)
        assert not np.isnan(radf[live]).any() and (rad[live] > 0).all()
    finally:
        f64.close()


def test_oracle_clamp_zero_colour_is_not_clamped():
    """The fp32 oracle (the reference's arithmetic without contraction) on clamp_zero: colour exactly +0, clamped 0."""
    cloud, cam, groups = _scene()
    f = O.forward_from(cloud, cam, f32=True, render=False)
    try:
        g = groups["clamp_zero"]
        assert (f.radii[g] > 0).all() and (f.rgb[g] == 0).all() and (f.clamped[g] == 0).all()
    finally:
        f.close()


def _single(scale):
    cam = synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 64, 48, fovy_deg=50.0)
    cloud = synth.Cloud(np.zeros((1, 3), np.float32), np.full((1, 3), scale, np.float32),
                        np.array([[1, 0, 0, 0]], np.float32), np.array([[0.5]], np.float32),
                        np.full((1, 1, 3), 1.0, np.float32), 0)
    return cloud, cam


@pytest.mark.parametrize("f32", [False, True], ids=["fp64", "fp32"])
def test_oracle_saturates_the_radius(f32):
    """One isotropic Gaussian at the origin, 64x48, camera at z = -3.5: scale 1e18 gives radius INT_MAX and the whole
    4 x 3 grid (a host (int) cast gave INT_MIN and an inverted rectangle), scale 1e-30 the dilation's radius 3, and
    scale 1e7 a radius beyond 2^24 that still converts exactly."""
    cloud, cam = _single(1e18)
    f = O.forward_from(cloud, cam, f32=f32)
    assert f.radii[0] == INT_MAX and f.tiles_touched[0] == 12 and f.num_rendered == 12
    assert f.ranges[:, 1].tolist() == list(range(1, 13)) and (f.n_contrib == 1).all()
    f.close()
    cloud, cam = _single(1e-30)
    f = O.forward_from(cloud, cam, f32=f32)
    assert f.radii[0] == 3 and f.tiles_touched[0] == 2
    f.close()
    cloud, cam = _single(1e7)
    f = O.forward_from(cloud, cam, f32=f32)
    assert 4.4e8 < f.radii[0] < 4.42e8 and f.tiles_touched[0] == 12
    f.close()


@pytest.mark.parametrize("f32", [False, True], ids=["fp64", "fp32"])
def test_rectangles_inside_the_grid_and_R_small(f32):
    """From the oracle's forward state, before anything is launched: every visible Gaussian's rectangle has rmin <= rmax
    inside the grid, its tile count is the rectangle's area, and R is far below any capacity limit."""
    cloud, cam, _ = _scene()
    gx, gy = _grid(cam)
    f = O.forward_from(cloud, cam, f32=f32, render=False)
    try:
        vis = f.radii > 0
        x0, y0, x1, y1 = _rects(f.means2D, f.radii, gx, gy)
        assert ((x0 <= x1) & (y0 <= y1) & (x1 <= gx) & (y1 <= gy))[vis].all()
        assert np.array_equal(((x1 - x0) * (y1 - y0))[vis], f.tiles_touched[vis].astype(np.int64))
        assert f.num_rendered == int(f.tiles_touched.sum()) < 100_000
        assert (f.tiles_touched[f.radii == INT_MAX] == gx * gy).all() and (f.radii == INT_MAX).sum() >= 20
    finally:
        f.close()


def test_host_tile_rect_saturates(tmp_path_factory):
    """csrc/common.cuh's tile_rect built for the host (tests/emission_slot_host.cpp): a radius of INT_MAX and a centre
    far off the frame give the device's rectangles."""
    from test_sharded_deterministic import _slot_lib
    lib = _slot_lib(str(tmp_path_factory.mktemp("slot")))
    px = np.array([100.0, -1e12, 3e9, 50.0], np.float32)
    py = np.array([60.0, 20.0, -7e9, 30.0], np.float32)
    r = np.array([INT_MAX, INT_MAX, INT_MAX, 16777218], np.int32)
    out = np.zeros(4, np.uint32)
    gx, gy = 20, 13
    lib.owned_counts(4, px.ctypes.data, py.ctypes.data, r.ctypes.data, gx, gy, 1, 0, out.ctypes.data)
    x0, y0, x1, y1 = _rects(np.stack([px, py], 1), r, gx, gy)
    assert out.tolist() == ((x1 - x0) * (y1 - y0)).tolist() == [gx * gy, 0, 0, gx * gy]


def test_subblock_predicate_misses_nothing():
    """oracle/subblock_check over every (pixel, splat) pair of the scene's records as the kernels compute them (NaN and
    inf conics, conics of 1e3 and more, denormal opacities): no pair the blend would take is rejected."""
    from oracle import subblock_check
    cloud, cam, _ = _scene()
    f = synth.preprocess_fp32(cloud, cam)
    co = np.concatenate([f["conic"], cloud.opacities], 1)
    c = subblock_check.scene(f["means2D"], co, f["radius"].astype(np.int32), cam.image_width, cam.image_height)
    assert c["misses"] == 0 and c["hits"] > 0 and c["blocks"] > 0, c


@pytest.mark.parametrize("kind,factor", [("scale", s) for s in SCALES] + [("translate", t) for t in SHIFTS])
def test_rescaled_patch_straddles_the_near_cut(kind, factor):
    """The Gaussians straight in front of the eye fall on both sides of the near cut at every factor, the patch stays in
    view, and the translated camera sits factor units from the origin."""
    cloud, cam = synth.rescaled_patch(kind, factor)
    f = O.forward_from(cloud, cam, f32=False, render=False)
    try:
        V = cam.viewmatrix.astype(np.float64).T
        z = cloud.means3D[-50:].astype(np.float64) @ V[2, :3] + V[2, 3]
        assert ((z > 0) & (z <= 0.2)).sum() >= 3 and (z > 0.2).sum() >= 3, np.sort(z)
        assert (f.radii > 0).sum() >= 10
        if kind == "translate":
            assert np.linalg.norm(cam.campos) > 0.9 * factor
    finally:
        f.close()


# ---------------------------------------------------------------------------------------------------------------- GPU
def _fwd_fields(cloud, cam, colors_precomp=None):
    from test_parity_gpu import _ours_forward_fields
    return _ours_forward_fields(run_ours(cloud, cam, BG, colors_precomp=colors_precomp))


@pytest.mark.gpu
def test_forward_bit_exact_every_variant():
    """Every forward output bit for bit the reference's, under every render_fwd variant and both binning and depth-sort
    variants; radii and tile counts as synth.preprocess_fp32 restates the kernels."""
    from test_parity_gpu import FWD_EXACT, _Ref, _options, _ref_forward_fields, _ref_run
    cloud, cam, groups = _scene()
    ref = _Ref("magnitudes/fwd", lambda: _ref_forward_fields(_ref_run(cloud, cam, BG)), golden=GOLDEN)
    fields = FWD_EXACT + ("tiles_touched",)
    runs = [dict(render_fwd_variant=v) for v in range(6)]
    runs += [dict(binning_variant=b, depth_sort_variant=d) for b in (0, 1) for d in (0, 1)]
    for opts in runs:
        with _options(**opts):
            ours = _fwd_fields(cloud, cam)
        bad = [k for k in fields if not ref.equal(k, ours[k])]
        assert not bad, (opts, bad)
    radii = ours["radii"].cpu().numpy()
    want = synth.preprocess_fp32(cloud, cam)["radius"]
    assert np.array_equal(radii, want), np.flatnonzero(radii != want)
    assert (radii[groups["radius_edge"]] == [16777215, 16777216, 16777218, 2147483520] + [INT_MAX] * 4).all()
    gx, gy = _grid(cam)
    tt = ours["tiles_touched"].cpu().numpy()
    assert (tt[radii == INT_MAX] == gx * gy).all() and ours["R"] == int(tt.sum())
    col = ours["color"].cpu().numpy()
    assert np.isfinite(col).all() and np.isfinite(ours["depth"].cpu().numpy()).all()


def _dL(cam, seed=47):
    return np.random.default_rng(seed).uniform(-1, 1, size=(3, cam.image_height, cam.image_width)).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("deterministic", [False, True], ids=["default", "deterministic"])
def test_backward_against_reference(deterministic):
    """The colour backward against the reference's: non-finite entries at the same positions, finite entries to
    1e-4 + 10x the reference's run-to-run noise + 1.5x its distance from ours' fp64-finite groups; deterministic mode
    gives the same bits twice."""
    from test_deterministic_truth import _run
    from test_parity_gpu import GRAD_PAIRS, _Ref, _ref_run
    cloud, cam, groups = _scene()
    gC = _dL(cam)
    got, _ = _run(cloud, cam, BG, gC, deterministic=deterministic)
    if deterministic:
        again, _ = _run(cloud, cam, BG, gC, deterministic=True)
        for k in got:
            assert np.array_equal(got[k].view(np.int32), again[k].view(np.int32)), k

    def compute():
        r1, r2 = _ref_run(cloud, cam, BG, dL=gC), _ref_run(cloud, cam, BG, dL=gC)
        out = {}
        for _, b in GRAD_PAIRS:
            g1, g2 = r1["grads"][b].cpu().numpy(), r2["grads"][b].cpu().numpy()
            fin = np.isfinite(g1)
            out[b] = g1
            out["nonfinite/" + b] = np.flatnonzero(~fin)
            out["noise/" + b] = rel_l2(np.where(fin, g2, 0), np.where(fin, g1, 0))
        return out
    ref = _Ref("magnitudes/bwd", compute, close=[b for _, b in GRAD_PAIRS],
               full=["nonfinite/" + b for _, b in GRAD_PAIRS], golden=GOLDEN)
    nonfinite = 0
    for a, b in GRAD_PAIRS:
        g = got[a]
        bad = np.flatnonzero(~np.isfinite(g.ravel()))
        assert np.array_equal(bad, np.asarray(ref.value("nonfinite/" + b)).ravel()), (a, bad[:8])
        nonfinite += bad.size
        o, r = ref.pair(b, g)
        fin = np.isfinite(o) & np.isfinite(r)
        err = rel_l2(o[fin], r[fin])
        print(a, f"{err:.2e}", "noise", f"{ref.scalar('noise/' + b):.2e}", "non-finite", bad.size)
        assert err <= 1e-4 + 10 * ref.scalar("noise/" + b), (a, err)
    assert nonfinite > 0      # the NaN-conic splats that blend take NaN gradients in both builds


_FORMS = ["colour", "depth", "alpha"]


@pytest.mark.gpu
@pytest.mark.parametrize("deterministic", [False, True], ids=["default", "deterministic"])
@pytest.mark.parametrize("form", _FORMS)
def test_finite_groups_against_fp64(form, deterministic):
    """The colour, colour + depth and colour + alpha losses on the groups whose intermediates stay finite (opacity and
    colour extremes, vanishing scales) against the fp64 oracle, to max(5e-5, 2 d32) with d32 the fp32 oracle's own
    distance (test_camera_models._check)."""
    from test_camera_models import _check
    from test_deterministic_truth import _run, _truth, _upstreams
    cloud, cam = _finite_scene()
    gC, gD = _upstreams(cam, 53)
    got, _ = _run(cloud, cam, BG, gC, gD=gD if form == "depth" else None, gA=gC[0] if form == "alpha" else None,
                  deterministic=deterministic)
    truth = _truth(cloud, cam, BG, form, gC, gD)
    truth32 = _truth(cloud, cam, BG, form, gC, gD, f32=True)
    _check(got, truth, truth32, (form, deterministic))


def _patch_errors(kind, factor):
    """(errors of the deterministic colour backward from fp64, the fp32 oracle's errors from fp64) per gradient."""
    from test_camera_grad_truth import _matched
    from test_deterministic_truth import _run, _truth, _truth_errors, _upstreams
    cloud, cam = synth.rescaled_patch(kind, factor)
    far = np.linalg.norm(cloud.means3D.astype(np.float64) - cam.campos, axis=1) >= 0.05 * factor
    cloud = _matched(_sub(cloud, np.flatnonzero(far)), cam)[0]
    gC, _ = _upstreams(cam, 57)
    got, _ = _run(cloud, cam, BG, gC, deterministic=True)
    truth = _truth(cloud, cam, BG, "colour", gC, None)
    t32 = _truth(cloud, cam, BG, "colour", gC, None, f32=True)
    errs = _truth_errors(got, truth)
    return errs, _truth_errors({k: np.asarray(t32[k]).reshape(np.shape(got[k])) for k in errs}, truth)


@pytest.mark.gpu
@pytest.mark.parametrize("factor", SCALES)
def test_rescaled_patch_against_fp64(factor):
    """The patch scaled with its camera: every gradient's relative error from fp64 within twice the unscaled patch's
    own error + 1e-6, or within twice the fp32 oracle's (the reference's arithmetic) distance on the scaled patch where
    that is larger. Gaussians closer to the eye than 0.05 x factor are left out: at 1e2 and 1e4 their world coordinates
    of ~1e3 .. 1e5 carry an fp32 rounding that is a visible part of their view depth (measured on an H100 with them
    kept: dmean3D 0.13 from fp64 at 1e4, the fp32 oracle 0.11), digits any fp32 rasterizer loses."""
    base, _ = _patch_errors("scale", 1.0)
    errs, d32 = _patch_errors("scale", factor)
    bound = {k: max(2 * base[k] + 1e-6, 2 * d32[k]) for k in errs}
    print(factor, {k: f"{errs[k]:.2e} (unscaled {base[k]:.2e}, fp32 {d32[k]:.2e})" for k in errs})
    bad = {k: (errs[k], bound[k]) for k in errs if not errs[k] <= bound[k]}
    assert not bad, (factor, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("shift", SHIFTS)
def test_translated_patch_matches_reference(shift):
    """The patch and its camera translated by up to 1e5: every forward output bit for bit the reference's."""
    from test_parity_gpu import FWD_EXACT, _Ref, _ref_forward_fields, _ref_run
    cloud, cam = synth.rescaled_patch("translate", shift)
    ref = _Ref(f"magnitudes/translate/{shift:g}", lambda: _ref_forward_fields(_ref_run(cloud, cam, BG)), golden=GOLDEN)
    ours = _fwd_fields(cloud, cam)
    bad = [k for k in FWD_EXACT if not ref.equal(k, ours[k])]
    assert not bad, (shift, bad)
    assert ours["R"] > 0


@pytest.mark.gpu
def test_mark_visible_and_apply_weights_bit_exact():
    """markVisible bit for bit; apply_weights with masks in multiples of 2^-8 (every sum exact in fp32 in any order),
    default and deterministic, bit for bit the reference's."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    from oracle import ref_cuda
    from test_camera_models import _apply_weights
    from test_deterministic_truth import _aw_gpu, _dyadic_mask
    from test_parity_gpu import _Ref
    cloud, cam, _ = _scene()
    P = cloud.means3D.shape[0]
    ct = cloud_tensors(cloud, "cuda")
    rs = settings_from(cam, BG, cloud.sh_degree, "cuda")
    vis = GaussianRasterizer(rs).markVisible(ct["means3D"])
    mask = _dyadic_mask(2, cam.image_height, cam.image_width, seed=59)
    w0, c0 = _aw_gpu(cloud, cam, mask, False)
    w1, c1 = _aw_gpu(cloud, cam, mask, True)
    assert torch.equal(c0, c1) and torch.equal(w0.view(torch.int32), w1.view(torch.int32))

    def compute():
        R = ref_cuda.ReferenceRasterizer()
        out = {"visible": R.mark_visible(ct["means3D"], rs.viewmatrix, rs.projmatrix)}
        out["weights"], out["cnt"] = _apply_weights(R, ct, P, mask, rs)
        return out
    ref = _Ref("magnitudes/trace", compute, golden=GOLDEN)
    assert ref.equal("visible", vis) and ref.equal("cnt", c0) and ref.equal("weights", w0)
    assert int((c0 > 0).sum()) > 20


@pytest.mark.gpu
def test_static_capacity_at_R():
    """Static capacity equal to R: the default forward and backward bit for bit, status [R, 0]."""
    from test_static_capacity import _run as static_run, _upstream
    cloud, cam, _ = _scene()
    dev = torch.device("cuda")
    rs = settings_from(cam, BG, cloud.sh_degree, dev)
    up = _upstream(cam, dev)
    ref_out, ref_g, _ = static_run(rs, cloud, False, (), True, None, dev, up)
    R = int(run_ours(cloud, cam, BG)["R"])
    out, g, rast = static_run(rs, cloud, False, (), True, R, dev, up)
    assert rast.status.tolist() == [R, 0]
    bits = lambda t: t.view(torch.int32) if t.dtype == torch.float32 else t
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(out, ref_out))
    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(g, ref_g))


@pytest.mark.gpu
def test_grad_mask():
    """grad_mask (deterministic): edited rows equal the unmasked deterministic gradients bit for bit, the others +0.0."""
    from test_grad_mask import _check_masked
    cloud, cam, _ = _scene()
    m = np.random.default_rng(61).uniform(size=cloud.means3D.shape[0]) < 0.4
    _check_masked(cloud, cam, "sh", torch.from_numpy(m).cuda())


# isotropic splats (vanishing, radius_edge, overflow) under random rotations: their rotation gradient is zero in exact
# arithmetic and rounding noise here, as in test_tile_grid
_SKIP_ROT = ("drot",)


@pytest.mark.gpu
def test_sharded_paths_match_single_gpu():
    """Dense and sparse virtual ranks at world 2 (test_sharded's harness) against the single GPU: frames, depth, radii
    and R bit for bit, gradients to summation order (the rotation gradient, rounding noise on the isotropic splats,
    aside). The harness compares gradients by relative L2, so the splats with a NaN conic (whose NaN gradients
    test_backward_against_reference pins) are left out of the cloud, and so are the cancel_tiny and cancel_negative
    needles: their covariance gradient scales the conic gradient by 1 / det^2 of a rounding-decided det, so the order
    of the per-pixel sums alone moves their mean gradient by more than its size (test_backward_against_reference holds
    them to the reference's own run-to-run noise). The upstream is positive: under a signed one the colour gradient of
    an sh_1e30 splat cancels, and its rounding, scaled by coefficients of 1e30, would decide the relative error."""
    from test_sharded import virtual_dense, virtual_sparse
    cloud, cam, _ = _scene()
    gC = np.random.default_rng(63).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    _, _, groups = _scene()
    keep = ~np.isnan(synth.preprocess_fp32(cloud, cam)["conic"]).any(1)
    assert 5 <= (~keep).sum() <= 20
    keep[np.concatenate([groups["cancel_tiny"], groups["cancel_negative"]])] = False
    cloud = _sub(cloud, np.flatnonzero(keep))
    case = dict(cloud=cloud, cam=cam, bg=BG, dL=gC, ref=run_ours(cloud, cam, bg=BG, dL=gC))
    virtual_dense(case, 2, skip=_SKIP_ROT)
    virtual_sparse(case, 2, "tight", max_fill=1.0, skip=_SKIP_ROT)
