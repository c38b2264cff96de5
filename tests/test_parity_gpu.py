"""GPU parity tests (``pytest -m gpu``). Everything goes through the public
GaussianRasterizer API -> ctypes -> C ABI (include/gsr_b200.h) -> sm_90a kernels.

Checkers (test infrastructure only):
  * oracle/_ref/libdgr_ref.so -- the reference's own CUDA sources compiled unmodified: integer outputs
    (radii, R, tile ranges, sorted point list, n_contrib) must be BIT-EXACT, images bit-exact, gradients to
    tolerance (the reference's float atomics are themselves order-dependent). Where that library is not built, every
    test compares against values recorded from it by tools/make_golden.py under tests/golden/parity/: SHA-256 digests
    of what must be bit-exact, short arrays in full, and a seeded sample of every array compared to a tolerance;
  * oracle/liboracle_cpu.so -- the CPU restatement (fp32 mirror and fp64 truth).
Tolerances are the ones SURVEY.md 8(a) fixes.
"""
import hashlib
import os

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import synth, _lib
from oracle import cpu_oracle, ref_cuda
from util import run_ours, rel_l2, cloud_tensors, settings_from

pytestmark = pytest.mark.gpu


def _ref_run(cloud, cam, bg, dL=None, colors_precomp=None, scale_modifier=1.0):
    dev = "cuda"
    ct = cloud_tensors(cloud, dev)
    rs = settings_from(cam, bg, cloud.sh_degree, dev, scale_modifier)
    R = ref_cuda.ReferenceRasterizer()
    cp = None if colors_precomp is None else torch.from_numpy(colors_precomp).to(dev)
    common = dict(means3D=ct["means3D"], shs=None if cp is not None else ct["shs"], colors_precomp=cp,
                  scales=ct["scales"], rotations=ct["rotations"], cov3D_precomp=None, bg=rs.bg,
                  viewmatrix=rs.viewmatrix, projmatrix=rs.projmatrix, campos=rs.campos, tanfovx=rs.tanfovx,
                  tanfovy=rs.tanfovy, sh_degree=cloud.sh_degree, scale_modifier=scale_modifier)
    color, radii, depth, nr = R.forward(opacities=ct["opacities"], image_height=cam.image_height,
                                        image_width=cam.image_width, **common)
    out = dict(color=color, radii=radii, depth=depth, R=nr, state=R.state())
    if dL is not None:
        out["grads"] = R.backward(dL_dcolor=torch.from_numpy(dL).to(dev), radii=radii, R=nr, **common)
    torch.cuda.synchronize()
    return out


SMALL_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "parity", "small_cases_reference.npz")
GRAD_PAIRS = [("dmean3D", "dL_dmeans3D"), ("dmean2D", "dL_dmeans2D"), ("dopacity", "dL_dopacity"),
              ("dscale", "dL_dscales"), ("drot", "dL_drotations"), ("dsh", "dL_dsh")]


def _digest(t):
    """SHA-256 of an array's values (integers as int64, floats as float32) and shape: equal digests = equal arrays."""
    a = t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
    a = np.ascontiguousarray(a.astype(np.float32 if a.dtype.kind == "f" else np.int64))
    return hashlib.sha256(str(a.shape).encode() + a.tobytes()).hexdigest()


def _ours_forward_fields(ours):
    v = ours["views"]
    vis = ours["radii"] > 0
    rec = v["records"][vis]
    return dict(R=ours["R"], radii=ours["radii"], tiles_touched=v["tiles_touched"], ranges=v["ranges"],
                point_list=v["point_list"], n_contrib=v["n_contrib"], final_T=v["final_T"], color=ours["color"],
                depth=ours["depth"], means2D=rec[:, 0:2], conic_opacity=rec[:, [2, 3, 4, 5]], depths=rec[:, 6],
                rgb=rec[:, 8:11])


def _ref_forward_fields(ref):
    s = ref["state"]
    vis = ref["radii"] > 0
    return dict(R=ref["R"], radii=ref["radii"], tiles_touched=s["tiles_touched"], ranges=s["ranges"],
                point_list=s["point_list"], n_contrib=s["n_contrib"], final_T=s["final_T"], color=ref["color"],
                depth=ref["depth"], means2D=s["means2D"][vis], conic_opacity=s["conic_opacity"][vis],
                depths=s["depths"][vis], rgb=s["rgb"][vis])


def _small_case_dL(cam):
    return np.random.default_rng(7).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)


def _small_golden():
    if not os.path.exists(SMALL_GOLDEN):
        pytest.fail("tests/golden/parity/small_cases_reference.npz missing (tools/make_golden.py writes it)")
    return np.load(SMALL_GOLDEN)


REF_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "parity", "reference_outputs.npz")
REF_SAMPLE = 1024
RECORD = None   # tools/make_golden.py sets a dict here: every reference value a _Ref computes is recorded into it


def _canon(x):
    """numpy array of a tensor / array / number: floats as float32, integers and booleans as int64."""
    a = x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    return np.ascontiguousarray(a.astype(np.float32 if a.dtype.kind == "f" else np.int64))


class _Ref:
    """The reference's values for one test case: computed by ``compute()`` from oracle/_ref when it is built, otherwise
    read from tests/golden/parity/reference_outputs.npz (recorded from it by tools/make_golden.py). Recorded per value:
    its SHA-256 digest (bit-exact checks), size and max |value|; the value itself when it has at most 64 entries or is
    named in ``full``; a seeded sample of REF_SAMPLE entries when it is named in ``close`` (compared to a tolerance).
    ``golden``: the recorded file to read."""

    def __init__(self, key, compute, close=(), full=(), golden=REF_GOLDEN):
        self.key = key
        self.live = ref_cuda.available()
        if self.live:
            self.v = {k: _canon(x) for k, x in compute().items()}
            if RECORD is not None:
                for k, a in self.v.items():
                    RECORD[f"{key}/{k}#digest"] = np.array(_digest(a))
                    RECORD[f"{key}/{k}#size"] = np.int64(a.size)
                    RECORD[f"{key}/{k}#absmax"] = np.float64(np.abs(a).max() if a.size else 0.0)
                    if a.size <= 64 or k in full:
                        RECORD[f"{key}/{k}"] = a
                    elif k in close:
                        RECORD[f"{key}/{k}#sample"] = a.ravel()[_sample_index(a.size)]
        else:
            if not os.path.exists(golden):
                pytest.fail(f"{os.path.relpath(golden)} missing (tools/make_golden.py writes it)")
            self.z = np.load(golden)
            if f"{key}/" not in {k[:len(key) + 1] for k in self.z.files}:
                pytest.fail(f"no recorded reference values for {key}")

    def equal(self, name, ours):
        """ours == the reference's value, bit for bit (same shape, same values)."""
        want = _digest(self.v[name]) if self.live else str(self.z[f"{self.key}/{name}#digest"])
        return _digest(ours) == want

    def value(self, name):
        """A small value (scalar or short array) of the reference, exactly."""
        return self.v[name] if self.live else self.z[f"{self.key}/{name}"]

    def scalar(self, name):
        return self.value(name).item()

    def pair(self, name, ours):
        """(ours, reference) as flat arrays: complete where the reference array is at hand, else on the recorded sample."""
        o = _canon(ours).ravel()
        if self.live:
            return o, self.v[name].ravel()
        k = f"{self.key}/{name}"
        assert o.size == int(self.z[k + "#size"]), (k, o.size)
        if k in self.z.files:
            return o, self.z[k].ravel()
        return o[_sample_index(o.size)], self.z[k + "#sample"]

    def absmax(self, name):
        return float(np.abs(self.v[name]).max()) if self.live else float(self.z[f"{self.key}/{name}#absmax"])


def _sample_index(n, size=REF_SAMPLE):
    return np.sort(np.random.default_rng(0).choice(n, size=min(n, size), replace=False))


def _small_cases():
    c1, cams1 = synth.make_config("c1")
    c3, cams3 = synth.make_config("c3", P=60_000)
    cam3 = synth.ring_cameras(8, 4.5, 15.0, 400, 304, 61.0)[2]   # H not a multiple of 16*? 304 = 19*16; W 400 = 25*16
    cam_odd = synth.ring_cameras(8, 4.5, 15.0, 333, 201, 61.0)[5]  # partial last tile row and column
    return [("c1", c1, cams1[0], (0.0, 0.0, 0.0)), ("c3s", c3, cam3, (1.0, 1.0, 1.0)),
            ("c3odd", c3, cam_odd, (0.2, 0.5, 0.7))]


@pytest.mark.parametrize("fwd_variant", [0, 1, 2, 3, 4, 5])
def test_forward_matches_reference_cuda_bit_exact(fwd_variant):
    live = ref_cuda.available()
    gold = None if live else _small_golden()
    with _options(render_fwd_variant=fwd_variant):
        for name, cloud, cam, bg in _small_cases():
            ours = _ours_forward_fields(run_ours(cloud, cam, bg))
            if live:
                want = {k: _digest(x) for k, x in _ref_forward_fields(_ref_run(cloud, cam, bg)).items()}
            else:
                want = {k: str(gold[f"{name}/fwd/{k}"]) for k in ours}
            for k, x in ours.items():
                assert _digest(x) == want[k], (name, k)


@pytest.mark.parametrize("bwd_variant", [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14])
def test_backward_matches_reference_cuda(bwd_variant):
    live = ref_cuda.available()
    gold = None if live else _small_golden()
    with _options(render_bwd_variant=bwd_variant):
        for name, cloud, cam, bg in _small_cases():
            dL = _small_case_dL(cam)
            ours = run_ours(cloud, cam, bg, dL=dL)
            if live:
                ref = _ref_run(cloud, cam, bg, dL=dL)
                ref2 = _ref_run(cloud, cam, bg, dL=dL)  # the reference's own run-to-run noise floor
            for a, b in GRAD_PAIRS:
                g = ours["grads"][a].cpu().numpy().ravel()
                if live:
                    r = ref["grads"][b].cpu().numpy().ravel()
                    noise = rel_l2(ref2["grads"][b].cpu().numpy().ravel(), r)
                    rmax = np.abs(r).max()
                else:   # the stored sample of the reference's gradient, its noise floor and its max over all entries
                    g = g[_sample_index(g.size)]
                    r = gold[f"{name}/bwd/{b}"]
                    noise, rmax = float(gold[f"{name}/bwd/{b}/noise"]), float(gold[f"{name}/bwd/{b}/absmax"])
                err = rel_l2(g, r)
                assert err <= 1e-4 + 10 * noise, (name, a, err, noise)
                assert np.abs(g - r).max() <= 1e-3 * rmax + 1e-12, (name, a)


def test_forward_backward_vs_cpu_oracle():
    for name, cloud, cam, bg in _small_cases()[:2]:
        rng = np.random.default_rng(3)
        dL = rng.uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
        ours = run_ours(cloud, cam, bg, dL=dL)
        f = cpu_oracle.forward_from(cloud, cam, bg)
        radii = ours["radii"].cpu().numpy()
        # FMA contraction on the GPU vs none on the CPU: allow <= 1e-4 of the Gaussians to differ by a radius step
        assert (radii != f.radii).mean() <= 1e-4, name
        tiles = ours["views"]["tiles_touched"].cpu().numpy().astype(np.uint32)
        assert (tiles != f.tiles_touched).mean() <= 1e-4, name
        if np.array_equal(radii, f.radii) and np.array_equal(tiles, f.tiles_touched):
            assert ours["R"] == f.num_rendered
            assert np.array_equal(ours["views"]["ranges"].cpu().numpy().astype(np.uint32), f.ranges)
        col = ours["color"].cpu().numpy()
        assert np.mean(np.abs(col - f.color) > 1e-5 + 1e-4 * np.abs(f.color)) <= 1e-4, name
        g = f.backward(dL)
        for a, b in [("dmean3D", "dmean3D"), ("dmean2D", "dmean2D"), ("dopacity", "dopacity"), ("dscale", "dscale"),
                     ("drot", "drot"), ("dsh", "dsh")]:
            assert rel_l2(ours["grads"][a].cpu().numpy(), g[b]) <= 2e-4, (name, a)
        f.close()


def test_precomputed_colors_and_scale_modifier():
    cloud, cams = synth.make_config("c2", P=20_000)
    cam = synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 320, 240, fovy_deg=50.0)
    rng = np.random.default_rng(11)
    cp = rng.uniform(size=(cloud.means3D.shape[0], 3)).astype(np.float32)
    dL = rng.uniform(size=(3, 240, 320)).astype(np.float32)
    ours = run_ours(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp, scale_modifier=0.7)

    def compute():
        ref = _ref_run(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp, scale_modifier=0.7)
        return dict(radii=ref["radii"], color=ref["color"], dL_dcolors=ref["grads"]["dL_dcolors"],
                    dL_dmeans3D=ref["grads"]["dL_dmeans3D"])
    ref = _Ref("precomputed_colors", compute, close=("dL_dcolors", "dL_dmeans3D"))
    assert ref.equal("radii", ours["radii"])
    assert ref.equal("color", ours["color"])
    assert rel_l2(*ref.pair("dL_dcolors", ours["grads"]["dcolor"])) <= 1e-4
    assert rel_l2(*ref.pair("dL_dmeans3D", ours["grads"]["dmean3D"])) <= 1e-4


def test_edge_cases_empty_and_all_culled():
    dev = "cuda"
    cam = synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 64, 48, fovy_deg=50.0)
    empty = synth.Cloud(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros((0, 4), np.float32),
                        np.zeros((0, 1), np.float32), np.zeros((0, 1, 3), np.float32), 0)
    out = run_ours(empty, cam, (0.3, 0.2, 0.1))
    assert out["R"] == 0 and out["color"].abs().sum().item() == 0.0  # rasterize_points.cu:72: outputs stay zero
    # every Gaussian behind the camera -> background only, zero gradients
    c, _ = synth.make_config("c1", P=500)
    c.means3D[:, 2] = -10.0
    dL = np.ones((3, 48, 64), np.float32)
    out = run_ours(c, cam, (0.3, 0.2, 0.1), dL=dL)
    assert out["R"] == 0 and int((out["radii"] > 0).sum()) == 0
    assert torch.allclose(out["color"][0], torch.full((48, 64), 0.3, device=dev))
    for k, g in out["grads"].items():
        if g is not None:
            assert float(g.abs().sum()) == 0.0, k


def test_mark_visible_and_apply_weights_match_reference():
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    cloud, cams = synth.make_config("c3", P=30_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 256, 192, 61.0)[1]
    ct = cloud_tensors(cloud, dev)
    rs = settings_from(cam, (0, 0, 0), 0, dev)
    rast = GaussianRasterizer(rs)
    vis = rast.markVisible(ct["means3D"])
    P = ct["means3D"].shape[0]
    rng = np.random.default_rng(5)
    mask = torch.from_numpy((rng.uniform(size=(1, 192, 256)) > 0.5).astype(np.float32)).to(dev)
    w1 = torch.zeros(P, 1, device=dev); c1 = torch.zeros(P, 1, dtype=torch.int32, device=dev)
    rast.apply_weights(ct["means3D"], None, ct["opacities"], None, w1, ct["scales"], ct["rotations"], None, c1, mask)
    torch.cuda.synchronize()

    def compute():
        R = ref_cuda.ReferenceRasterizer()
        w2 = torch.zeros(P, 1, device=dev); c2 = torch.zeros(P, 1, dtype=torch.int32, device=dev)
        R.apply_weights(means3D=ct["means3D"], opacities=ct["opacities"], scales=ct["scales"], rotations=ct["rotations"],
                        weights=w2, cnt=c2, image_weights=mask, bg=rs.bg, viewmatrix=rs.viewmatrix,
                        projmatrix=rs.projmatrix, campos=rs.campos, tanfovx=rs.tanfovx, tanfovy=rs.tanfovy,
                        image_height=192, image_width=256)
        torch.cuda.synchronize()
        return dict(visible=R.mark_visible(ct["means3D"], rs.viewmatrix, rs.projmatrix), cnt=c2, weights=w2)
    ref = _Ref("mark_visible_apply_weights", compute)
    assert ref.equal("visible", vis)
    assert ref.equal("cnt", c1)
    assert ref.equal("weights", w1)  # mask values are 0/1 -> sums are exact integers in fp32


@pytest.mark.parametrize("CH,binary", [(1, False), (2, True), (2, False), (3, True), (3, False)])
def test_apply_weights_channels_and_float_masks(CH, binary):
    """apply_weights for CH = 1..3 (cuda_rasterizer/apply_weights.cu:365-380) and non-binary masks: `cnt` advances by
    CH per (pixel, splat) hit (:331-334) and must be EXACT; `weights` are float sums in a different order than the
    reference's per-hit atomics: exact for 0/1 masks (integer sums), <= 1e-5 relative for float masks."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    cloud, _ = synth.make_config("c3", P=25_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 333, 201, 61.0)[CH]      # partial last tile row and column
    H, W = cam.image_height, cam.image_width
    ct = cloud_tensors(cloud, dev)
    rs = settings_from(cam, (0, 0, 0), 0, dev)
    P = ct["means3D"].shape[0]
    rng = np.random.default_rng(17 + CH)
    m = rng.uniform(size=(CH, H, W)).astype(np.float32)
    if binary:
        m = (m > 0.4).astype(np.float32)
    mask = torch.from_numpy(m).to(dev)
    w1 = torch.zeros(P, CH, device=dev); c1 = torch.zeros(P, 1, dtype=torch.int32, device=dev)
    GaussianRasterizer(rs).apply_weights(ct["means3D"], None, ct["opacities"], None, w1, ct["scales"], ct["rotations"],
                                         None, c1, mask)
    torch.cuda.synchronize()

    def compute():
        w2 = torch.zeros(P, CH, device=dev); c2 = torch.zeros(P, 1, dtype=torch.int32, device=dev)
        ref_cuda.ReferenceRasterizer().apply_weights(
            means3D=ct["means3D"], opacities=ct["opacities"], scales=ct["scales"], rotations=ct["rotations"], weights=w2,
            cnt=c2, image_weights=mask, bg=rs.bg, viewmatrix=rs.viewmatrix, projmatrix=rs.projmatrix, campos=rs.campos,
            tanfovx=rs.tanfovx, tanfovy=rs.tanfovy, image_height=H, image_width=W)
        torch.cuda.synchronize()
        return dict(cnt=c2, cnt_sum=int(c2.sum()), weights=w2)
    ref = _Ref(f"apply_weights/{CH}/{binary}", compute, close=("weights",))
    cnt_sum = ref.scalar("cnt_sum")
    assert cnt_sum > 0 and cnt_sum % CH == 0
    assert ref.equal("cnt", c1)
    if binary:
        assert ref.equal("weights", w1)
    else:
        g, r = ref.pair("weights", w1)
        assert rel_l2(g, r) <= 1e-5
        assert np.abs(g - r).max() <= 1e-4 * ref.absmax("weights")
    # a second call ACCUMULATES (the reference never zeroes weights / cnt: rasterize_points.cu:223-231)
    c_once = c1.clone()
    GaussianRasterizer(rs).apply_weights(ct["means3D"], None, ct["opacities"], None, w1, ct["scales"], ct["rotations"],
                                         None, c1, mask)
    assert torch.equal(c1, 2 * c_once)


def test_alpha_output_matches_reference_accum_alpha_and_is_differentiable():
    """Opt-in alpha image (north star: RGB / depth / alpha): alpha = 1 - final_T must equal 1 - the reference's
    ImageState::accum_alpha bit for bit; its gradient is checked through the identity
        color_0 with bg = (-1, 0, 0)  ==  C_0 - T_final  ==  C_0 + alpha - 1,
    i.e. d/dtheta [ sum G*(color_0 | bg=0) + sum G*alpha ] == d/dtheta sum G*(color_0 | bg=(-1,0,0))."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    cloud, _ = synth.make_config("c3", P=40_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 333, 201, 61.0)[2]
    H, W = cam.image_height, cam.image_width
    G = torch.from_numpy(np.random.default_rng(23).uniform(size=(H, W)).astype(np.float32)).to(dev)

    def run(bg, with_alpha):
        ct = cloud_tensors(cloud, dev, requires_grad=True)
        m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
        rs = settings_from(cam, bg, cloud.sh_degree, dev)
        out = GaussianRasterizer(rs, return_alpha=with_alpha)(means3D=ct["means3D"], means2D=m2, opacities=ct["opacities"],
                                                              shs=ct["shs"], scales=ct["scales"], rotations=ct["rotations"])
        loss = (out[0][0] * G).sum()
        if with_alpha:
            assert len(out) == 4 and out[3].shape == (1, H, W)
            loss = loss + (out[3][0] * G).sum()
        loss.backward()
        grads = {k: v.grad.detach().cpu().numpy() for k, v in ct.items()}
        grads["means2D"] = m2.grad.detach().cpu().numpy()
        return out, grads

    out_a, g_a = run((0.0, 0.0, 0.0), True)

    def compute():
        ref = _ref_run(cloud, cam, (0.0, 0.0, 0.0))
        return dict(alpha=1.0 - ref["state"]["final_T"], color=ref["color"])
    ref = _Ref("alpha", compute)
    assert ref.equal("alpha", out_a[3][0].detach())
    assert ref.equal("color", out_a[0].detach())
    out_b, g_b = run((-1.0, 0.0, 0.0), False)
    assert len(out_b) == 3
    for k in g_a:
        assert rel_l2(g_a[k], g_b[k]) <= 2e-5, (k, rel_l2(g_a[k], g_b[k]))


def test_camera_gradients_match_the_fp64_oracle_chain_and_finite_differences():
    """North star: backward over {..., viewmatrix}. The reference has no camera gradient, so the check is first
    principles, in three layers:
      1. tests/test_camera_grad_math.py (CPU): the formulas equal autograd of the smooth per-Gaussian forward map (1e-9);
      2. here: the CUDA kernel equals those formulas evaluated in float64 on the fp64 CPU oracle's upstream gradients
         (dL/dmean2D, dL/dconic, dL/dcolour of the same scene and loss), rel. L2 <= 1e-3 for all three camera arrays;
      3. here: viewmatrix and campos also agree with CENTRAL FINITE DIFFERENCES of the oracle's forward within 6 %.
         The pipeline is discontinuous where a pixel crosses a splat's alpha = 1/255 contour, the T < 1e-4 cut or the
         3-sigma tile rectangle, and the analytic gradient (the reference's, for every parameter) ignores the motion of
         those edges while a finite difference integrates it: the fp64 differences themselves move by 2-7 % between
         step sizes for the view matrix, and by far more for the projection matrix (210 / 188 / 24 / 68 for entry
         [0,0] at h = 2^-7 / 2^-11 / 2^-13 / 2^-15 against 243.7 analytic), which is why projmatrix has no layer 3."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    from test_camera_grad_math import camera_grads_formulas
    dev = "cuda"
    cloud, _ = synth.make_config("c3", P=4000)
    cloud.shs = np.ascontiguousarray(cloud.shs[:, :4, :])      # degree 1: what camera_grads_formulas restates
    cloud.sh_degree = 1
    cam = synth.ring_cameras(8, 4.5, 15.0, 96, 64, 61.0)[3]
    H, W = cam.image_height, cam.image_width
    bg = (0.2, 0.1, 0.3)
    G = np.random.default_rng(31).uniform(0.5, 1.5, size=(3, H, W)).astype(np.float32)
    ct = cloud_tensors(cloud, dev)
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    view = rs.viewmatrix.clone().requires_grad_(True)
    proj = rs.projmatrix.clone().requires_grad_(True)
    cpos = rs.campos.clone().requires_grad_(True)
    rs = rs._replace(viewmatrix=view, projmatrix=proj, campos=cpos)
    out = GaussianRasterizer(rs, camera_grad=True)(means3D=ct["means3D"], means2D=torch.zeros_like(ct["means3D"]),
                                                   opacities=ct["opacities"], shs=ct["shs"], scales=ct["scales"],
                                                   rotations=ct["rotations"])
    (out[0] * torch.from_numpy(G).to(dev)).sum().backward()
    got = dict(viewmatrix=view.grad.cpu().numpy().astype(np.float64), projmatrix=proj.grad.cpu().numpy().astype(np.float64),
               campos=cpos.grad.cpu().numpy().astype(np.float64))
    assert np.all(got["viewmatrix"][:, 3] == 0) and np.all(got["projmatrix"][:, 2] == 0)   # entries the forward never reads

    # layer 2: the chain rule in float64 on the oracle's upstream gradients
    f = cpu_oracle.forward_from(cloud, cam, bg, f32=False)
    g = f.backward(G)
    vis = f.radii > 0
    hx, hy = W / (2 * cam.tanfovx), H / (2 * cam.tanfovy)
    t = (cloud.means3D[vis].astype(np.float64) @ cam.viewmatrix.astype(np.float64)[:3, :3]) + cam.viewmatrix.astype(np.float64)[3, :3]
    assert np.all(np.abs(t[:, 0] / t[:, 2]) < 1.3 * cam.tanfovx) and np.all(np.abs(t[:, 1] / t[:, 2]) < 1.3 * cam.tanfovy)  # nobody clamped
    g_conic = np.stack([g["dconic"][vis, 0, 0], g["dconic"][vis, 0, 1], g["dconic"][vis, 1, 1]], 1)
    g_col = g["dcolor"][vis] * (1.0 - f.clamped[vis].astype(np.float64))
    dv, dp, dc = camera_grads_formulas(cam.viewmatrix.astype(np.float64), cam.projmatrix.astype(np.float64),
                                       cam.campos.astype(np.float64), cloud.means3D[vis].astype(np.float64),
                                       f.cov3D[vis].astype(np.float64), cloud.shs[vis].astype(np.float64),
                                       g["dmean2D"][vis, :2], g_conic, g_col, hx, hy)
    f.close()
    for name, want in (("viewmatrix", dv), ("projmatrix", dp), ("campos", dc)):
        assert rel_l2(got[name], want) <= 1e-3, (name, rel_l2(got[name], want), got[name], want)

    # layer 3: finite differences of the fp64 forward (float32-representable steps) for the two stable arrays
    def loss(**over):
        ff = cpu_oracle.forward_from(cloud, cam, bg, f32=False, **over)
        v = float((ff.color * G).sum())
        ff.close()
        return v
    h = np.float32(2.0 ** -11)
    for name, arr in (("viewmatrix", cam.viewmatrix.astype(np.float32)), ("campos", cam.campos.astype(np.float32))):
        fd = np.zeros(arr.shape, np.float64)
        for idx in np.ndindex(arr.shape):
            if name == "viewmatrix" and idx[1] == 3:
                continue
            ap, am = arr.copy(), arr.copy()
            ap[idx] += h; am[idx] -= h
            fd[idx] = (loss(**{name: ap}) - loss(**{name: am})) / float(ap[idx] - am[idx])
        assert np.linalg.norm(fd) > 0 and rel_l2(got[name], fd) <= 6e-2, (name, rel_l2(got[name], fd), got[name], fd)


def test_full_size_properties_config3():
    """BASELINE config 3 (1M Gaussians, 1600x1200): size-independent properties at full size."""
    cloud, cams = synth.make_config("c3")
    cam = cams[0]
    dL = np.random.default_rng(1).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    out = run_ours(cloud, cam, (0, 0, 0), dL=dL)
    v = out["views"]
    R = out["R"]
    assert R == int(v["tiles_touched"].sum())
    ranges = v["ranges"].cpu().numpy().astype(np.int64)
    nz = ranges[ranges[:, 1] > ranges[:, 0]]
    assert nz[:, 1].max() == R and int((nz[:, 1] - nz[:, 0]).sum()) == R   # ranges tile the list exactly
    keys = v["tile_keys"].cpu().numpy()
    if keys.dtype == np.int16:
        keys = keys.view(np.uint16)
    assert np.all(np.diff(keys.astype(np.int64)) >= 0)                       # sorted by tile
    pl = v["point_list"].cpu().numpy()
    depth = v["records"][:, 6].cpu().numpy()
    d = depth[pl]
    same_tile = keys[1:] == keys[:-1]
    assert np.all(d[1:][same_tile] >= d[:-1][same_tile])                     # depth-sorted inside every tile
    tie = same_tile & (d[1:] == d[:-1])
    assert np.all(pl[1:][tie] > pl[:-1][tie])                                # stable: ties by Gaussian index
    assert np.array_equal(np.bincount(pl, minlength=cloud.means3D.shape[0]), v["tiles_touched"].cpu().numpy())
    col = out["color"]
    assert torch.isfinite(col).all() and float(col.min()) >= 0.0
    T = v["final_T"]
    assert float(T.min()) >= float(np.float32(1e-4)) and float(T.max()) <= 1.0
    vis = (out["radii"] > 0)
    for k, g in out["grads"].items():
        if g is None:
            continue
        assert torch.isfinite(g).all(), k
        assert float(g[~vis].abs().sum()) == 0.0, k                          # culled Gaussians get exact zeros
    # linearity of the backward in dL/dpixel
    out2 = run_ours(cloud, cam, (0, 0, 0), dL=2.0 * dL)
    a, b = out["grads"]["dmean3D"], out2["grads"]["dmean3D"]
    assert rel_l2((2 * a).cpu().numpy(), b.cpu().numpy()) <= 1e-4


def test_host_buffer_api():
    """C-ABI host-buffer entry points (gsr_host_*): same images as the tensor path, checksums of all gradients."""
    import ctypes as C
    lib = _lib.load()
    cloud, _ = synth.make_config("c3", P=50_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 320, 240, 61.0)[4]
    dL = np.random.default_rng(2).uniform(size=(3, 240, 320)).astype(np.float32)
    ref = run_ours(cloud, cam, (0.2, 0.3, 0.4), dL=dL)
    ctx = C.c_void_p(lib.gsr_host_create())
    assert ctx.value
    P, M = cloud.means3D.shape[0], cloud.shs.shape[1]
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    arrs = [np.ascontiguousarray(x, np.float32) for x in (cloud.means3D, cloud.opacities, cloud.shs, cloud.scales, cloud.rotations)]
    _lib.check(lib.gsr_host_upload_cloud(ctx, P, M, *[p(a) for a in arrs]), "upload")
    bg = np.array([0.2, 0.3, 0.4], np.float32)
    s = _lib.Settings(240, 320, cam.tanfovx, cam.tanfovy, 1.0, 3, M, 0, 0, p(bg).value, p(cam.viewmatrix).value,
                      p(cam.projmatrix).value, p(cam.campos).value)
    color = np.zeros((3, 240, 320), np.float32); radii = np.zeros(P, np.int32); sums = np.zeros(8, np.float64)
    R = lib.gsr_host_step(ctx, C.byref(s), p(dL), p(color), p(radii), p(sums))
    lib.gsr_host_destroy(ctx)
    assert R == ref["R"]
    assert np.array_equal(color, ref["color"].cpu().numpy())
    assert np.array_equal(radii, ref["radii"].cpu().numpy())
    g = ref["grads"]
    want = [g["dmean3D"], g["dmean2D"], None, g["dopacity"], None, g["dsh"], g["dscale"], g["drot"]]
    for i, w in enumerate(want):
        if w is not None:
            ws = float(w.double().sum())
            scale = float(w.double().abs().sum()) + 1e-12
            assert abs(sums[i] - ws) <= 1e-5 * scale, (i, sums[i], ws)


def test_speculative_second_half_equals_exact_path():
    """The sync-free forward (capacity guessed from the previous frame) must give the same bits as the exact path,
    including when the guess is too small and the second half is redone."""
    import gaussianeditor_b200.rasterizer as RZ
    cloud, _ = synth.make_config("c3", P=40_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 320, 240, 61.0)[6]
    dL = np.random.default_rng(9).uniform(size=(3, 240, 320)).astype(np.float32)
    key = (0, cloud.means3D.shape[0], 320, 240)
    try:
        RZ.SPECULATIVE = False
        exact = run_ours(cloud, cam, (0.5, 0.5, 0.5), dL=dL)
        RZ.SPECULATIVE = True
        RZ._r_hint[key] = exact["R"]            # good guess -> speculative path
        spec = run_ours(cloud, cam, (0.5, 0.5, 0.5), dL=dL)
        assert spec["state"].cap > spec["R"] == exact["R"]
        RZ._r_hint[key] = 10                    # hopeless guess -> overflow -> redo with the exact size
        redo = run_ours(cloud, cam, (0.5, 0.5, 0.5), dL=dL)
        assert redo["state"].cap == redo["R"] == exact["R"]
        for other in (spec, redo):
            assert torch.equal(other["color"], exact["color"]) and torch.equal(other["depth"], exact["depth"])
            assert torch.equal(other["views"]["point_list"], exact["views"]["point_list"])
            assert torch.equal(other["views"]["ranges"], exact["views"]["ranges"])
            assert torch.equal(other["views"]["n_contrib"], exact["views"]["n_contrib"])
            for k in ("dmean3D", "dsh", "dopacity"):
                assert rel_l2(other["grads"][k].cpu().numpy(), exact["grads"][k].cpu().numpy()) <= 1e-5
    finally:
        RZ.SPECULATIVE = True


@pytest.mark.parametrize("variant,depth_variant", [(0, 0), (1, 1), (1, 0), (0, 1)])
def test_binning_variants_match_reference_lists(variant, depth_variant):
    """Both binning implementations -- 0: emit kernel + CUB radix sort + tile_ranges (binning.cu), 1: difference-array
    ranges + two own radix passes with the emission fused in (tile_binning.cu, default) -- and both depth orders -- 0: CUB
    radix sort + CUB scan (default), 1: depth_sort.cu -- must give the reference's point_list / ranges / R bit for bit,
    incl. a partial last tile row/column and a frame with > 256 tile columns."""
    with _options(binning_variant=variant, depth_sort_variant=depth_variant):
        cloud, _ = synth.make_config("c3", P=80_000)
        for (W, H, k) in [(333, 201, 5), (4160, 48, 1), (1600, 1200, 2)]:
            cam = synth.ring_cameras(8, 4.5, 15.0, W, H, 61.0)[k]
            ours = run_ours(cloud, cam, (0.1, 0.2, 0.3))

            def compute():
                ref = _ref_run(cloud, cam, (0.1, 0.2, 0.3))
                s = ref["state"]
                return dict(R=ref["R"], ranges=s["ranges"], point_list=s["point_list"], color=ref["color"])
            ref = _Ref(f"binning/{W}x{H}", compute)
            v = ours["views"]
            assert ours["R"] == ref.scalar("R"), (W, H)
            assert ref.equal("ranges", v["ranges"]), (W, H)
            assert ref.equal("point_list", v["point_list"]), (W, H)
            assert ref.equal("color", ours["color"]), (W, H)


def test_depth_order_and_offsets_equal_cub_at_full_size():
    """depth_sort.cu against the CUB sort + scan it replaces, at BASELINE config 3 size (1M keys, 39 % of them the
    culled key 0xFFFFFFFF, ties between equal depths): depth_order and the instance total must be identical."""
    from gaussianeditor_b200.rasterizer import forward_state_views
    cloud, cams = synth.make_config("c3")
    res = {}
    for v in (0, 1):
        with _options(depth_sort_variant=v):
            out = run_ours(cloud, cams[2], (0, 0, 0))
        res[v] = (out["views"]["depth_order"].clone(), out["R"], out["views"]["point_list"].clone())
    vis = int((out["radii"] > 0).sum())
    assert torch.equal(res[0][0][:vis], res[1][0][:vis])       # among the culled (equal keys) both are index-ordered too:
    assert torch.equal(res[0][0], res[1][0])
    assert res[0][1] == res[1][1] and torch.equal(res[0][2], res[1][2])


def test_edit_loop_harness_runs_and_densifies():
    """Config-5 loop shape (2 forwards + 1 backward per step, densification changing P) on a small cloud."""
    from gaussianeditor_b200 import edit_loop
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    out = edit_loop.run_edit_loop(GaussianRasterizer, steps=8, P=20_000, densification_interval=3)
    assert out["P_last"] != out["P_first"] and 0.0 < out["render_fraction"] < 1.0
    assert np.isfinite(out["final_loss"])


def test_edit_loop_matches_the_reference_rasterizer_step_by_step():
    """SURVEY 8(f-2): the SAME config-5-shaped loop (two renders + one backward per step, Adam, densify / prune
    changing P) driven once by this repository's rasterizer and once by the reference's own CUDA kernels
    (oracle/ref_torch.RefGaussianRasterizer) from identical seeds: the Gaussian count after every densification must be
    identical, the loss trajectories must agree to 1e-3, and the max_radii2D bookkeeping (what the reference's prune
    test reads) must be identical at the first densification and agree on >= 99.9 % of the Gaussians at the end.
    Ours runs in deterministic mode: 20 Adam steps amplify the last-bit differences of the default backward's float
    atomics, and its end-of-loop max_radii2D agreement moved between 1.0 and 0.99898 from run to run (H100)."""
    import functools
    from gaussianeditor_b200 import edit_loop
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    kw = dict(steps=20, P=20_000, densification_interval=5, seed=3)
    det = functools.partial(GaussianRasterizer, deterministic=True)
    ours = edit_loop.run_edit_loop(det, **kw)

    def compute():
        from oracle.ref_torch import RefGaussianRasterizer
        ref = edit_loop.run_edit_loop(RefGaussianRasterizer, **kw)
        return dict(counts=np.array(ref["counts"]), losses=np.array(ref["losses"]),
                    max_radii2D_first=ref["max_radii2D_at_densify"][0], max_radii2D=ref["max_radii2D"])
    ref = _Ref("edit_loop", compute, full=("counts", "losses", "max_radii2D"))
    counts = [int(c) for c in ref.value("counts")]
    assert ours["counts"] == counts and len(set(ours["counts"])) >= 3       # P changed, identically
    lo, lr = np.array(ours["losses"]), np.asarray(ref.value("losses"), np.float64)
    assert np.all(np.isfinite(lo)) and np.abs(lo - lr).max() <= 1e-3 * np.abs(lr).max(), np.abs(lo - lr).max()
    assert ref.equal("max_radii2D_first", ours["max_radii2D_at_densify"][0])
    mine, theirs = ref.pair("max_radii2D", ours["max_radii2D"])
    same = float((mine == theirs).mean())
    assert same >= 0.999, same
    # the fused-activation entry point must drive the same loop to the same counts
    fused = edit_loop.run_edit_loop(det, fused_activations=True, **kw)
    assert fused["counts"] == counts
    assert np.abs(np.array(fused["losses"]) - lr).max() <= 1e-3 * np.abs(lr).max()


@pytest.mark.parametrize("deg,M", [(0, 16), (1, 16), (2, 16), (3, 16), (1, 4), (2, 9), (0, 1)])
def test_sh_degrees_and_coefficient_counts(deg, M):
    """Active degree below the allocated one (GaussianEditor ramps sh_degree up), M = 4 / 16 take the TMA row path,
    M = 1 / 9 the plain-load path; coefficients above the active degree must get exactly zero gradient."""
    cloud, _ = synth.make_config("c3", P=30_000)
    cloud.shs = np.ascontiguousarray(cloud.shs[:, :M, :])
    cloud.sh_degree = deg
    cam = synth.ring_cameras(8, 4.5, 15.0, 208, 160, 61.0)[3]
    dL = np.random.default_rng(deg * 7 + M).uniform(size=(3, 160, 208)).astype(np.float32)
    ours = run_ours(cloud, cam, (0.1, 0.1, 0.1), dL=dL)

    def compute():
        ref = _ref_run(cloud, cam, (0.1, 0.1, 0.1), dL=dL)
        rv = ref["radii"] > 0
        rc = ref["state"]["clamped"][rv]
        g = ref["grads"]
        return dict(radii=ref["radii"], color=ref["color"], rgb=ref["state"]["rgb"][rv],
                    clamped=(rc[:, 0] + 2 * rc[:, 1] + 4 * rc[:, 2]).to(torch.uint8),
                    dL_dsh=g["dL_dsh"], dL_dmeans3D=g["dL_dmeans3D"], dL_dopacity=g["dL_dopacity"])
    ref = _Ref(f"sh/{deg}/{M}", compute, close=("dL_dsh", "dL_dmeans3D", "dL_dopacity"))
    assert ref.equal("radii", ours["radii"]) and ref.equal("color", ours["color"])
    vis = ours["radii"] > 0
    assert ref.equal("rgb", ours["views"]["records"][vis][:, 8:11])
    assert ref.equal("clamped", ours["views"]["clamped"][vis])
    for a, b in [("dsh", "dL_dsh"), ("dmean3D", "dL_dmeans3D"), ("dopacity", "dL_dopacity")]:
        err = rel_l2(*ref.pair(b, ours["grads"][a]))
        assert err <= 1e-4, ((deg, M), a, err)
    nb = (deg + 1) ** 2
    assert float(ours["grads"]["dsh"][:, nb:, :].abs().sum()) == 0.0


def test_precomputed_covariance_path():
    """cov3D_precomp instead of scale/rotation (unused by GaussianEditor but part of the API): forward bit-exact,
    dL/dcov3D to tolerance, scale/rotation gradients absent."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    cloud, _ = synth.make_config("c3", P=20_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 192, 144, 61.0)[5]
    f = cpu_oracle.forward_from(cloud, cam, render=False)          # cov3D from the oracle as the precomputed input
    cov = torch.from_numpy(f.cov3D.astype(np.float32)).to(dev).requires_grad_(True)
    f.close()
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    rs = settings_from(cam, (0, 0, 0), 3, dev)
    m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
    color, radii, depth = GaussianRasterizer(rs)(means3D=ct["means3D"], means2D=m2, opacities=ct["opacities"],
                                                 shs=ct["shs"], cov3D_precomp=cov)
    dL = torch.from_numpy(np.random.default_rng(13).uniform(size=(3, 144, 192)).astype(np.float32)).to(dev)
    (color * dL).sum().backward()

    def compute():
        R = ref_cuda.ReferenceRasterizer()
        common = dict(means3D=ct["means3D"].detach(), shs=ct["shs"].detach(), colors_precomp=None, scales=None,
                      rotations=None, cov3D_precomp=cov.detach(), bg=rs.bg, viewmatrix=rs.viewmatrix,
                      projmatrix=rs.projmatrix, campos=rs.campos, tanfovx=rs.tanfovx, tanfovy=rs.tanfovy, sh_degree=3)
        rc, rr, rd, n = R.forward(opacities=ct["opacities"].detach(), image_height=144, image_width=192, **common)
        g = R.backward(dL_dcolor=dL, radii=rr, R=n, **common)
        return dict(radii=rr, color=rc, dL_dcov3D=g["dL_dcov3D"], dL_dmeans3D=g["dL_dmeans3D"])
    ref = _Ref("precomputed_covariance", compute, close=("dL_dcov3D", "dL_dmeans3D"))
    assert ref.equal("radii", radii) and ref.equal("color", color.detach())
    assert rel_l2(*ref.pair("dL_dcov3D", cov.grad)) <= 1e-4
    assert rel_l2(*ref.pair("dL_dmeans3D", ct["means3D"].grad)) <= 1e-4


def test_hd_frame_partial_tile_row_and_debug_flag():
    """1920x1080: 1080 is not a multiple of 16 (68 tile rows, last partial); debug=True synchronises after each launch."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians, forward_state_views
    dev = "cuda"
    cloud, _ = synth.make_config("c3", P=150_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 1920, 1080, 61.0)[1]
    ct = cloud_tensors(cloud, dev)
    rs = settings_from(cam, (0.3, 0.6, 0.9), 3, dev, debug=True)
    color, radii, depth = GaussianRasterizer(rs)(means3D=ct["means3D"], means2D=torch.zeros_like(ct["means3D"]),
                                                 opacities=ct["opacities"], shs=ct["shs"], scales=ct["scales"],
                                                 rotations=ct["rotations"])
    v = forward_state_views(_RasterizeGaussians.last_state)

    def compute():
        ref = _ref_run(cloud, cam, (0.3, 0.6, 0.9))
        s = ref["state"]
        return dict(radii=ref["radii"], ranges=s["ranges"], color=ref["color"], depth=ref["depth"],
                    n_contrib=s["n_contrib"])
    ref = _Ref("hd_frame", compute)
    assert v["ranges"].shape[0] == 120 * 68
    assert ref.equal("radii", radii) and ref.equal("ranges", v["ranges"])
    assert ref.equal("color", color) and ref.equal("depth", depth)
    assert ref.equal("n_contrib", v["n_contrib"])


@pytest.mark.parametrize("cfg", ["c2", "c3"])
def test_full_size_configs_match_reference_cuda(cfg):
    """BASELINE configs 2 (100k, SH 0, 800x800) and 3 (1M, SH 3, 1600x1200) at FULL size against the reference's
    own CUDA build: forward bit-exact (images, radii, n_contrib, final_T, the complete sorted list).

    Gradients are judged against the fp64 CPU oracle (ground truth), because at full size the REFERENCE is the
    inaccurate one: its ~10^6 per-pixel fp32 atomics on the largest splats swamp small addends and under-count
    (config 3: reference 2.5e-4 .. 6.3e-4 relative L2 from fp64; this repo 1e-6 .. 1.3e-5, like the fp32 CPU oracle).
    So: ours vs fp64 <= 5e-5, and ours vs reference no further apart than the reference is from the truth."""
    cloud, cams = synth.make_config(cfg)
    cam = cams[-1]
    bg = (0.1, 0.2, 0.3)
    dL = np.random.default_rng(11).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    ours = run_ours(cloud, cam, bg, dL=dL)
    f64 = cpu_oracle.forward_from(cloud, cam, bg, f32=False)
    truth = f64.backward(dL)
    f64.close()
    pairs = [("dmean3D", "dL_dmeans3D"), ("dmean2D", "dL_dmeans2D"), ("dopacity", "dL_dopacity"),
             ("dscale", "dL_dscales"), ("drot", "dL_drotations"), ("dsh", "dL_dsh")]

    def compute():
        ref = _ref_run(cloud, cam, bg, dL=dL)
        ref2 = _ref_run(cloud, cam, bg, dL=dL)
        s = ref["state"]
        out = dict(R=ref["R"], radii=ref["radii"], color=ref["color"], depth=ref["depth"],
                   n_contrib=s["n_contrib"].flatten(), final_T=s["final_T"].flatten(), point_list=s["point_list"])
        for a, b in pairs:
            r = ref["grads"][b].cpu().numpy()
            out[b] = r
            out["noise/" + b] = rel_l2(ref2["grads"][b].cpu().numpy(), r)
            out["ref_err/" + b] = rel_l2(r, truth[a])
        return out
    ref = _Ref(f"full_size/{cfg}", compute, close=[b for _, b in pairs])
    v = ours["views"]
    assert ours["R"] == ref.scalar("R"), cfg
    for name, x in [("radii", ours["radii"]), ("color", ours["color"]), ("depth", ours["depth"]),
                    ("n_contrib", v["n_contrib"].flatten()), ("final_T", v["final_T"].flatten()),
                    ("point_list", v["point_list"])]:
        assert ref.equal(name, x), (cfg, name)
    for a, b in pairs:
        g, t = ours["grads"][a].cpu().numpy(), truth[a]
        noise, ref_err = ref.scalar("noise/" + b), ref.scalar("ref_err/" + b)
        ours_err = rel_l2(g, t)
        assert ours_err <= 5e-5, (cfg, a, ours_err)
        # the reference's own distance from the truth must stay inside a fixed band, so that a regression of OURS
        # cannot hide behind a growing ref_err term
        assert ref_err <= 1.5e-3, (cfg, a, ref_err)
        err = rel_l2(*ref.pair(b, g))
        assert err <= 1e-4 + 10 * noise + 1.5 * ref_err, (cfg, a, err, noise, ref_err)


def test_full_size_properties_config4():
    """BASELINE config 4 (5M Gaussians, 1920x1080) on one GPU: list invariants, determinism of the forward
    (bit-identical across two runs), finite gradients that vanish exactly for culled Gaussians."""
    cloud, cams = synth.make_config("c4")
    cam = cams[3]
    dL = np.random.default_rng(2).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    out = run_ours(cloud, cam, (0, 0, 0), dL=dL)
    v, R = out["views"], out["R"]
    assert R == int(v["tiles_touched"].to(torch.int64).sum())
    ranges = v["ranges"].to(torch.int64)
    lens = ranges[:, 1] - ranges[:, 0]
    assert int(lens.sum()) == R and int(lens.min()) >= 0 and int(ranges[:, 1].max()) == R
    keys = v["tile_keys"]
    keys = (keys.to(torch.int32) & 0xFFFF) if keys.dtype == torch.int16 else keys
    assert bool((keys[1:] >= keys[:-1]).all())
    pl = v["point_list"].to(torch.int64)
    d = v["records"][:, 6][pl]
    same = keys[1:] == keys[:-1]
    assert bool((d[1:][same] >= d[:-1][same]).all())
    tie = same & (d[1:] == d[:-1])
    assert bool((pl[1:][tie] > pl[:-1][tie]).all())
    assert float(v["final_T"].min()) >= float(np.float32(1e-4)) and float(v["final_T"].max()) <= 1.0
    vis = out["radii"] > 0
    for k, g in out["grads"].items():
        if g is not None:
            assert torch.isfinite(g).all(), k
            assert float(g[~vis].abs().sum()) == 0.0, k
    again = run_ours(cloud, cam, (0, 0, 0))
    assert torch.equal(again["color"], out["color"]) and torch.equal(again["radii"], out["radii"])
    assert torch.equal(again["views"]["point_list"], v["point_list"]) and again["R"] == R


def _raw_params(cloud, dev, seed=0):
    """Inverse activations of a synth.Cloud -> leaf tensors shaped like the scene model's raw parameters
    (scene/gaussian_model.py:_xyz, _features_dc, _features_rest, _opacity, _scaling, _rotation)."""
    g = torch.Generator().manual_seed(seed)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    op = t(cloud.opacities).clamp(1e-6, 1 - 1e-6)
    rot = t(cloud.rotations) * (0.25 + 3.0 * torch.rand(cloud.rotations.shape[0], 1, generator=g)).to(dev)  # unnormalised
    raw = dict(xyz=t(cloud.means3D), opacity=torch.log(op / (1 - op)), features_dc=t(cloud.shs[:, :1, :]),
               features_rest=t(cloud.shs[:, 1:, :]), scaling=torch.log(t(cloud.scales)), rotation=rot)
    return {k: v.contiguous().requires_grad_(True) for k, v in raw.items()}


@pytest.mark.parametrize("deg,M,P", [(3, 16, 60013), (3, 16, 4096), (1, 4, 20000), (0, 1, 5000)])
def test_fused_activations_match_pytorch_prologue(deg, M, P):
    """SURVEY 8(f-3): GaussianRasterizer.forward_raw (sigmoid / exp / normalize / SH concatenation inside the
    preprocess kernels) against the scene model's PyTorch prologue followed by the default rasterizer, forward and
    all raw-parameter gradients. P = 60013 ends in a partial block (plain-load fallback), 4096 is all bulk copies."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = torch.device("cuda")
    cloud, cams = synth.make_config("c3", P=P)
    cloud.shs = np.ascontiguousarray(cloud.shs[:, :M, :])
    cloud.sh_degree = deg
    cam = synth.ring_cameras(8, 4.5, 15.0, 640, 400, 61.0)[1]
    rs = settings_from(cam, (0.3, 0.1, 0.2), deg, dev)
    dL = torch.from_numpy(np.random.default_rng(5).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)).to(dev)
    rast = GaussianRasterizer(rs)

    a = _raw_params(cloud, dev)
    m2a = torch.zeros_like(a["xyz"], requires_grad=True)
    col_a, rad_a, dep_a = rast(means3D=a["xyz"], means2D=m2a, opacities=torch.sigmoid(a["opacity"]),
                               shs=torch.cat((a["features_dc"], a["features_rest"]), dim=1),
                               scales=torch.exp(a["scaling"]), rotations=torch.nn.functional.normalize(a["rotation"]))
    (col_a * dL).sum().backward()

    b = _raw_params(cloud, dev)
    m2b = torch.zeros_like(b["xyz"], requires_grad=True)
    col_b, rad_b, dep_b = rast.forward_raw(means3D=b["xyz"], means2D=m2b, opacity_logits=b["opacity"],
                                           features_dc=b["features_dc"], features_rest=b["features_rest"],
                                           log_scales=b["scaling"], raw_rotations=b["rotation"])
    (col_b * dL).sum().backward()

    assert float((rad_a != rad_b).float().mean()) <= 1e-4           # activations round differently in rare cases
    ca, cb = col_a.detach().cpu().numpy(), col_b.detach().cpu().numpy()
    assert np.mean(np.abs(ca - cb) > 1e-5 + 1e-4 * np.abs(ca)) <= 1e-4
    assert rel_l2(dep_b.detach().cpu().numpy(), dep_a.detach().cpu().numpy()) <= 1e-5
    same = (rad_a == rad_b)
    for k in a:
        ga, gb = a[k].grad, b[k].grad
        assert gb is not None and gb.shape == ga.shape, k
        assert torch.isfinite(gb).all(), k
        assert rel_l2(gb[same].cpu().numpy(), ga[same].cpu().numpy()) <= 1e-4, (k, rel_l2(gb[same].cpu().numpy(), ga[same].cpu().numpy()))
    assert rel_l2(m2b.grad[same].cpu().numpy(), m2a.grad[same].cpu().numpy()) <= 1e-4
    assert float(b["features_rest"].grad[rad_b == 0].abs().sum()) == 0.0   # culled rows are written as exact zeros


def test_blending_weights_conserve_energy_at_full_size():
    """Size-independent property at BASELINE config 3 size: with precomputed colours and dL/dpixel = 1 on one channel,
    dL/dcolor_i is the total blending weight of splat i, and the weights of all splats plus the remaining
    transmittance of every pixel add up to the number of pixels (sum_i alpha_i T_i + T_final = 1 per pixel)."""
    cloud, cams = synth.make_config("c3")
    cam = cams[5]
    H, W = cam.image_height, cam.image_width
    dL = np.zeros((3, H, W), np.float32)
    dL[1] = 1.0
    cols = np.random.default_rng(4).random((cloud.means3D.shape[0], 3), dtype=np.float32)
    out = run_ours(cloud, cam, (0.0, 0.0, 0.0), dL=dL, colors_precomp=cols)
    w = out["grads"]["dcolor"].double()
    assert float(w.min()) >= 0.0 and float(w[:, 0].abs().sum()) == 0.0 and float(w[:, 2].abs().sum()) == 0.0
    total = float(w[:, 1].sum()) + float(out["views"]["final_T"].double().sum())
    assert abs(total - H * W) <= 2e-5 * H * W, (total, H * W)


# ---- adversarial scenes and frame-size edges -----------------------------------------------------------------------

class _options:
    """Set rasterizer options for a block and restore the previous values afterwards (also on failure)."""

    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        lib = _lib.load()
        self.old = {k: int(lib.gsr_get_option(k.encode())) for k in self.kw}
        for k, v in self.kw.items():
            _lib.set_option(k, v)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            _lib.set_option(k, v)


FWD_EXACT = ("radii", "R", "ranges", "point_list", "n_contrib", "final_T", "color", "depth")


def _needle_case():
    cloud, cam = synth.needle_cloud()
    cp = np.random.default_rng(41).uniform(size=(cloud.means3D.shape[0], 3)).astype(np.float32)
    return cloud, cam, cp


@pytest.mark.parametrize("fwd_variant", [0, 1, 2, 3, 4, 5])
def test_needle_forward_bit_exact_every_variant(fwd_variant):
    """Needle splats (synth.needle_cloud: ~18 (pixel, splat) pairs that a threshold-relative culling margin would drop,
    tests/test_subblock_mask.py) must render bit-exact under every render_fwd variant. Variant 0 has no sub-block
    culling and is the control; variants 1-5 cull with csrc/common.cuh: splat_subblock_mask."""
    cloud, cam, cp = _needle_case()
    with _options(render_fwd_variant=fwd_variant):
        ours = _ours_forward_fields(run_ours(cloud, cam, (0, 0, 0), colors_precomp=cp))
    ref = _Ref("needle/fwd", lambda: _ref_forward_fields(_ref_run(cloud, cam, (0, 0, 0), colors_precomp=cp)))
    bad = [k for k in FWD_EXACT if not ref.equal(k, ours[k])]
    assert not bad, (fwd_variant, bad)


@pytest.mark.parametrize("bwd_variant", [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14])
def test_needle_backward_blend_weights_every_variant(bwd_variant):
    """Needle scene, precomputed colours, dL/dpixel = 1 on the green channel: dL/dcolor_i[1] is splat i's total blend
    weight, and one dropped (pixel, splat) hit moves it by alpha*T >= T/255. Compared per Gaussian with the reference's
    dL_dcolors to 3x its own run-to-run difference (float atomics) plus 1e-5 relative plus 1e-4 (fp32 sums of up to
    ~1e5 terms in another order than the reference's): below half a dropped hit for >= 75 % of the Gaussians.
    (The fp64 CPU oracle is no yardstick here: the fp32 conic of a needle, det = ac - b^2, is ill-conditioned, and the
    fp32 and fp64 gradients of dmean3D differ by a relative L2 of ~30.)"""
    cloud, cam, cp = _needle_case()
    H, W = cam.image_height, cam.image_width
    dL = np.zeros((3, H, W), np.float32)
    dL[1] = 1.0
    with _options(render_bwd_variant=bwd_variant):
        ours = run_ours(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp)

    def compute():
        a = _ref_run(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp)["grads"]["dL_dcolors"]
        b = _ref_run(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp)["grads"]["dL_dcolors"]
        return dict(dL_dcolors=a, noise=(a - b).abs())
    ref = _Ref("needle/bwd", compute, full=("dL_dcolors", "noise"))
    got = ours["grads"]["dcolor"].cpu().numpy().astype(np.float64)
    want = np.asarray(ref.value("dL_dcolors"), np.float64).reshape(got.shape)
    noise = np.asarray(ref.value("noise"), np.float64).reshape(got.shape)
    tol = 3.0 * noise + 1e-5 * np.abs(want) + 1e-4
    assert np.all(got[:, [0, 2]] == 0.0) and (want[:, 1] > 0.0).mean() > 0.9
    assert (tol[:, 1] < 0.5 / 255).mean() >= 0.75, np.percentile(tol[:, 1], [50, 90])   # sharp enough to see a dropped hit
    over = np.abs(got - want) > tol
    assert not over.any(), (bwd_variant, np.argwhere(over)[:8].tolist(), np.abs(got - want)[over][:8])


def _grads_vs_reference_and_truth(key, cloud, cam, bg, dL, ours, pairs, truth_tol):
    """ours vs the fp64 CPU oracle to truth_tol, and ours vs the reference to 1e-4 + 10x its run-to-run noise + 1.5x
    the reference's own distance from the fp64 oracle (its per-pixel fp32 atomics lose precision on large frames, see
    test_full_size_configs_match_reference_cuda), that distance itself bounded."""
    f64 = cpu_oracle.forward_from(cloud, cam, bg, f32=False)
    truth = f64.backward(dL)
    f64.close()

    def compute():
        r1 = _ref_run(cloud, cam, bg, dL=dL)
        r2 = _ref_run(cloud, cam, bg, dL=dL)
        out = dict(R=r1["R"], radii=r1["radii"], color=r1["color"], depth=r1["depth"])
        for a, b in pairs:
            out[b] = r1["grads"][b]
            out["noise/" + b] = rel_l2(r2["grads"][b].cpu().numpy(), r1["grads"][b].cpu().numpy())
            out["ref_err/" + b] = rel_l2(r1["grads"][b].cpu().numpy(), truth[a])
        return out
    ref = _Ref(key, compute, close=[b for _, b in pairs])
    assert ours["R"] == ref.scalar("R")
    for k in ("radii", "color", "depth"):
        assert ref.equal(k, ours[k]), (key, k)
    for a, b in pairs:
        g = ours["grads"][a].cpu().numpy()
        t = rel_l2(g, truth[a])
        assert t <= truth_tol, (key, a, t)
        ref_err = ref.scalar("ref_err/" + b)
        assert ref_err <= 1.5e-3, (key, a, ref_err)
        err = rel_l2(*ref.pair(b, g))
        assert err <= 1e-4 + 10 * ref.scalar("noise/" + b) + 1.5 * ref_err, (key, a, err, ref_err)


def test_frustum_edge_forward_and_preprocess_backward():
    """synth.frustum_edge_cloud: view depths at and around the 0.2 near cut, centres at the 1.3 tan(fov) Jacobian
    clamp, off-screen centres whose splat reaches the frame (SH row read without the bulk copy), splats larger than the
    frame, zero scale axes. Forward bit-exact under every render_fwd variant; all six gradients against the reference
    and the fp64 CPU oracle."""
    cloud, cam = synth.frustum_edge_cloud()
    bg = (0.1, 0.2, 0.3)
    dL = np.random.default_rng(43).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    for v in range(6):
        with _options(render_fwd_variant=v):
            fwd = _ours_forward_fields(run_ours(cloud, cam, bg))
        ref = _Ref("frustum_edge/fwd", lambda: _ref_forward_fields(_ref_run(cloud, cam, bg)))
        bad = [k for k in FWD_EXACT if not ref.equal(k, fwd[k])]
        assert not bad, (v, bad)
    ours = run_ours(cloud, cam, bg, dL=dL)
    _grads_vs_reference_and_truth("frustum_edge/bwd", cloud, cam, bg, dL, ours, GRAD_PAIRS, 5e-5)


def test_opacity_edge_forward_and_backward():
    """synth.opacity_edge_cloud: opacities at fp32(1/255) and its neighbours and at the 0.99 clamp, in stacks deep
    enough that the T < 1e-4 stop falls at varied list positions. Forward bit-exact under every render_fwd variant,
    backward under the CTA-per-tile and the default render_bwd variant."""
    cloud, cam = synth.opacity_edge_cloud()
    bg = (0.0, 0.5, 1.0)
    dL = np.random.default_rng(44).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    for v in range(6):
        with _options(render_fwd_variant=v):
            fwd = _ours_forward_fields(run_ours(cloud, cam, bg))
        ref = _Ref("opacity_edge/fwd", lambda: _ref_forward_fields(_ref_run(cloud, cam, bg)))
        bad = [k for k in FWD_EXACT if not ref.equal(k, fwd[k])]
        assert not bad, (v, bad)
    T = fwd["final_T"].cpu().numpy()
    assert T.min() < 1e-3            # some pixels reached the T < 1e-4 stop
    for v in (0, 14):
        with _options(render_bwd_variant=v):
            ours = run_ours(cloud, cam, bg, dL=dL)
        _grads_vs_reference_and_truth("opacity_edge/bwd", cloud, cam, bg, dL, ours, GRAD_PAIRS, 5e-5)


FRAME_SIZES = [(16, 16), (32, 16), (17, 9), (1, 1), (2048, 1536), (3840, 2160), (4112, 4096)]


@pytest.mark.parametrize("W,H,key_bits", [(w, h, 16) for w, h in FRAME_SIZES] + [(1600, 1200, 32)])
def test_frame_size_edges(W, H, key_bits):
    """Frame sizes the configs never use: single-tile and sub-tile frames (the single-digit copy of the tile sort),
    1x1, grids whose tile-count difference array does not fit in shared memory (2048x1536, 3840x2160: the global
    scratch path of tile_prefix with fewer replicas), 4112x4096 = 65792 tiles (the CUB fallback with 32-bit tile keys),
    and 1600x1200 with 32-bit tile keys forced. Forward bit-exact under both binning and both depth-sort variants,
    one backward against the reference and the fp64 CPU oracle."""
    cloud, _ = synth.make_config("c3", P=30_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, W, H, 61.0)[(W + H) % 8]
    bg = (0.3, 0.2, 0.1)
    key = f"frame/{W}x{H}/{key_bits}"
    ref = _Ref(key + "/fwd", lambda: _ref_forward_fields(_ref_run(cloud, cam, bg)))
    with _options(tile_key_bits=key_bits):
        for bv in (0, 1):
            for dv in (0, 1):
                with _options(binning_variant=bv, depth_sort_variant=dv):
                    fwd = _ours_forward_fields(run_ours(cloud, cam, bg))
                bad = [k for k in FWD_EXACT if not ref.equal(k, fwd[k])]
                assert not bad, (bv, dv, bad)
        assert fwd["ranges"].shape[0] == ((W + 15) // 16) * ((H + 15) // 16)
        dL = np.random.default_rng(45).uniform(size=(3, H, W)).astype(np.float32)
        ours = run_ours(cloud, cam, bg, dL=dL)
    pairs = [("dmean3D", "dL_dmeans3D"), ("dopacity", "dL_dopacity"), ("dsh", "dL_dsh")]
    _grads_vs_reference_and_truth(key + "/bwd", cloud, cam, bg, dL, ours, pairs, 5e-5)
