"""Opt-in depth gradient (``GaussianRasterizer(..., depth_grad=True)``, gsr_backward_depth / gsr_backward_raw_depth).

The depth image is D = sum_i z_i alpha_i T_i with no background term, i.e. a fourth colour channel with colour z_i and
background 0. The fp64 truth is built from the fp64 CPU oracle on exactly that identity (``depth_truth``): a second
oracle pass renders the colours (z_hi, z_lo, 1) with background 0 and upstream (dL/dD, dL/dD, dL/dA), where
z_hi + z_lo is the oracle's fp64 view depth split into two fp32 numbers (the oracle takes colours in fp32) and the
third channel sum_i alpha_i T_i = 1 - T_final is the alpha image. Its dL/dcolour_0 is dL/dz_i; the preprocess term
dL/dz * (V[2], V[6], V[10]) of the mean is added in float64. The CPU tests pin that construction against closed forms
and against torch autograd of the blend; the GPU tests hold the CUDA kernels to it.
"""
import numpy as np
import pytest
import torch

from gaussianeditor_b200 import synth
from oracle import cpu_oracle as O
from util import cloud_tensors, rel_l2, settings_from

C0 = 0.28209479177387814
A_MAX = float(np.float32(0.99))   # the alpha clamp 0.99f of the forward


# ---- the fp64 truth ------------------------------------------------------------------------------------------------

def _forward64(cloud, cam, bg, colors_precomp=None, cov3D_precomp=None, scale_modifier=1.0, f32=False):
    kw = dict(scale_modifier=scale_modifier)
    if colors_precomp is not None:
        kw["colors_precomp"] = colors_precomp
    if cov3D_precomp is not None:
        kw.update(cov3D_precomp=cov3D_precomp, scales=None, rotations=None)
    return O.forward_from(cloud, cam, bg, f32=f32, **kw)


def depth_truth(cloud, cam, bg, gC=None, gD=None, gA=None, colors_precomp=None, cov3D_precomp=None,
                scale_modifier=1.0, f32=False):
    """fp64 gradients of  sum gC*colour + sum gD*depth + sum gA*alpha  (each upstream optional). Returns the oracle's
    gradient dict plus ``ddepth`` [P] (dL/dz per Gaussian), and the colour-pass forward as ``fwd``. ``f32=True``: the
    same construction on the fp32 oracle (the reference's arithmetic), to measure how far fp32 lies from the truth."""
    f = _forward64(cloud, cam, bg, colors_precomp, cov3D_precomp, scale_modifier, f32)
    P, M, H, W = f.P, f.M, f.H, f.W
    if gC is not None:
        g = f.backward(np.asarray(gC, np.float32))
    else:
        g = dict(dmean2D=np.zeros((P, 3)), dconic=np.zeros((P, 2, 2)), dopacity=np.zeros((P, 1)),
                 dcolor=np.zeros((P, 3)), dmean3D=np.zeros((P, 3)), dcov3D=np.zeros((P, 6)),
                 dsh=np.zeros((P, M, 3)), dscale=np.zeros((P, 3)), drot=np.zeros((P, 4)))
    g["ddepth"] = np.zeros(P)
    if gD is not None or gA is not None:
        hi = f.depths.astype(np.float32)
        lo = (f.depths - hi.astype(np.float64)).astype(np.float32)
        cols = np.stack([hi, lo, np.ones(P, np.float32)], 1)
        fd = _forward64(cloud, cam, (0.0, 0.0, 0.0), cols, cov3D_precomp, scale_modifier, f32)
        assert np.array_equal(fd.n_contrib, f.n_contrib) and np.array_equal(fd.point_list, f.point_list)
        up = np.zeros((3, H, W), np.float32)
        if gD is not None:
            up[0] = up[1] = gD
        if gA is not None:
            up[2] = gA
        gd = fd.backward(up)
        fd.close()
        for k in ("dmean2D", "dconic", "dopacity", "dmean3D", "dcov3D", "dscale", "drot"):
            g[k] = g[k] + gd[k]
        if gD is not None:
            g["ddepth"] = gd["dcolor"][:, 0].copy()
            V = cam.viewmatrix.astype(np.float32).astype(np.float64).reshape(-1)
            g["dmean3D"] = g["dmean3D"] + g["ddepth"][:, None] * V[[2, 6, 10]][None, :]
    g["fwd"] = f
    return g


# ---- CPU: the construction ------------------------------------------------------------------------------------------

def _kat_scene():
    """The two-Gaussian scene of test_oracle_kat.py::test_two_gaussians_compositing_and_stop_rule."""
    cam = synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 32, 32, fovy_deg=50.0)
    s = 0.5
    sh = np.zeros((2, 1, 3), np.float32)
    sh[:, 0, :] = (np.array([[0, 1, 0], [1, 0, 0]], np.float32) - 0.5) / C0
    cloud = synth.Cloud(np.array([[0, 0, 1.0], [0, 0, -1.0]], np.float32), np.full((2, 3), s, np.float32),
                        np.array([[1, 0, 0, 0]] * 2, np.float32), np.array([[0.9], [0.6]], np.float32), sh, 0)
    return cloud, cam


def test_closed_form_two_gaussians():
    """D = z1*a1 + z0*(1-a1)*a0 at the centre pixel (z1 = 2.5 front, z0 = 4.5 back); with dL/dD one-hot there:
    dL/do1 = (z1 - z0*a0)*G1, dL/do0 = z0*(1-a1)*G0 (the 0.99 clamp passes the gradient, as in the reference),
    dL/dz1 = a1, dL/dz0 = (1-a1)*a0."""
    cloud, cam = _kat_scene()
    gD = np.zeros((32, 32), np.float32)
    py = px = 16
    gD[py, px] = 1.0
    g = depth_truth(cloud, cam, (0.0, 0.0, 0.0), gD=gD)
    f = g["fwd"]
    assert abs(f.depths[1] - 2.5) < 1e-6 and abs(f.depths[0] - 4.5) < 1e-6
    co = f.conic_opacity

    def gauss(i):
        dx, dy = f.means2D[i] - np.array([px, py], np.float64)
        return np.exp(-0.5 * (co[i, 0] * dx * dx + co[i, 2] * dy * dy) - co[i, 1] * dx * dy)
    G1, G0 = gauss(1), gauss(0)
    a1, a0 = min(A_MAX, co[1, 3] * G1), min(A_MAX, co[0, 3] * G0)
    z1, z0 = f.depths[1], f.depths[0]
    assert abs(f.depth[0, py, px] - (z1 * a1 + z0 * (1 - a1) * a0)) < 1e-9
    assert abs(g["dopacity"][1, 0] - (z1 - z0 * a0) * G1) < 1e-9
    assert abs(g["dopacity"][0, 0] - z0 * (1 - a1) * G0) < 1e-9
    assert abs(g["ddepth"][1] - a1) < 1e-9
    assert abs(g["ddepth"][0] - (1 - a1) * a0) < 1e-9
    f.close()


def _blend_autograd(f, bg, gC, gD):
    """The blend restated in torch float64 on the oracle's forward state (means2D, conic_opacity, rgb, depths,
    point_list, ranges) with the hit set frozen as the oracle decided it; returns autograd's gradients in the oracle's
    conventions (dmean2D in NDC units: x 0.5*W, y 0.5*H; dconic[0,1] = half of dL/db)."""
    H, W = f.H, f.W
    t = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    m2, con, rgb, z = t(f.means2D), t(f.conic_opacity[:, :3]), t(f.rgb), t(f.depths)
    op = t(f.conic_opacity[:, 3])
    gx = (W + 15) // 16
    loss = torch.zeros((), dtype=torch.float64)
    bgt = torch.tensor(np.asarray(bg, np.float32).astype(np.float64))   # the oracle reads bg as fp32
    for py in range(H):
        for px in range(W):
            tile = (py // 16) * gx + px // 16
            r0, r1 = f.ranges[tile]
            ids = f.point_list[r0:r0 + int(f.n_contrib[py, px])].astype(np.int64)
            if ids.size == 0:
                continue
            dx = f.means2D[ids, 0] - px
            dy = f.means2D[ids, 1] - py
            co = f.conic_opacity[ids]
            power = -0.5 * (co[:, 0] * dx * dx + co[:, 2] * dy * dy) - co[:, 1] * dx * dy
            alpha = np.minimum(A_MAX, co[:, 3] * np.exp(power))
            hit = (power <= 0) & (alpha >= np.float32(1.0 / 255.0))
            ids = torch.from_numpy(ids[hit])
            if ids.numel() == 0:
                continue
            DX, DY = m2[ids, 0] - px, m2[ids, 1] - py
            c = con[ids]
            G = torch.exp(-0.5 * (c[:, 0] * DX * DX + c[:, 2] * DY * DY) - c[:, 1] * DX * DY)
            a = op[ids] * G
            a = a - (a - A_MAX).clamp(min=0).detach()   # the 0.99 clamp without cutting the gradient (reference)
            T = torch.cumprod(torch.cat([torch.ones(1, dtype=torch.float64), 1 - a]), 0)
            w = a * T[:-1]
            C = (w[:, None] * rgb[ids]).sum(0) + T[-1] * bgt
            D = (w * z[ids]).sum()
            loss = loss + (C * torch.from_numpy(gC[:, py, px].astype(np.float64))).sum() + D * float(gD[py, px])
    loss.backward()
    dm = m2.grad.numpy() * np.array([0.5 * W, 0.5 * H])
    dcon = con.grad.numpy() * np.array([1.0, 0.5, 1.0])
    return dict(dmean2D=dm, dconic=dcon, dopacity=op.grad.numpy(), dcolor=rgb.grad.numpy(), ddepth=z.grad.numpy())


def test_blend_backward_matches_autograd():
    """300 Gaussians on 48x32 pixels (six tiles, many overlaps), colour and depth upstreams and a background."""
    cloud, cams = synth.make_config("c3", P=300)
    cloud.scales = (cloud.scales * 6.0).astype(np.float32)
    cam = synth.look_at_camera((0, 0.5, -4.0), (0, 0, 0), (0, -1, 0), 48, 32, fovy_deg=40.0)
    bg = (0.3, 0.2, 0.1)
    rng = np.random.default_rng(7)
    gC = rng.normal(size=(3, 32, 48)).astype(np.float32)
    gD = rng.normal(size=(32, 48)).astype(np.float32)
    g = depth_truth(cloud, cam, bg, gC=gC, gD=gD)
    f = g["fwd"]
    assert f.hits > 3 * 48 * 32, f.hits
    want = _blend_autograd(f, bg, gC, gD)
    got = dict(dmean2D=g["dmean2D"][:, :2], dconic=np.stack([g["dconic"][:, 0, 0], g["dconic"][:, 0, 1],
                                                             g["dconic"][:, 1, 1]], 1),
               dopacity=g["dopacity"][:, 0], dcolor=g["dcolor"], ddepth=g["ddepth"])
    for k in want:
        assert np.linalg.norm(want[k]) > 0, k
        assert rel_l2(got[k], want[k]) <= 1e-9, (k, rel_l2(got[k], want[k]))
    f.close()


def test_colour_only_oracle_path_unchanged():
    """Without a depth upstream the truth is the oracle's own backward: one forward, no depth pass, the same values.
    (Two oracle backward calls are equal only to fp64 rounding: its threads add the tiles' sums in the order they
    finish.)"""
    cloud, cams = synth.make_config("c3", P=300)
    cam = synth.look_at_camera((0, 0.5, -4.0), (0, 0, 0), (0, -1, 0), 48, 32, fovy_deg=40.0)
    gC = np.random.default_rng(8).uniform(size=(3, 32, 48)).astype(np.float32)
    f = _forward64(cloud, cam, (0.1, 0.2, 0.3))
    a = f.backward(gC)
    f.close()
    calls = []
    orig = O.forward_from
    O.forward_from = lambda *args, **kw: calls.append(1) or orig(*args, **kw)
    try:
        b = depth_truth(cloud, cam, (0.1, 0.2, 0.3), gC=gC)
    finally:
        O.forward_from = orig
    b["fwd"].close()
    assert len(calls) == 1
    for k in a:
        assert rel_l2(b[k], a[k]) <= 1e-13, k
    assert not b["ddepth"].any()


def test_render_constructs_the_rasterizer_as_the_reference_unless_asked():
    """render() builds its rasterizer with raster_settings only unless depth_grad=True: a class with the reference's
    constructor (as the edit-loop harness injects) keeps working, and depth_grad reaches the rasterizer when asked."""
    import types
    from gaussianeditor_b200 import gaussian_renderer as GR
    made = []

    class RefSignature:
        def __init__(self, raster_settings):
            made.append({})

        def __call__(self, **kw):
            P = kw["means3D"].shape[0]
            return torch.zeros(3, 4, 4), torch.ones(P, dtype=torch.int32), torch.zeros(1, 4, 4)

    class WithDepth(RefSignature):
        def __init__(self, raster_settings, depth_grad=False):
            made.append({"depth_grad": depth_grad})

    P = 5
    pc = types.SimpleNamespace(get_xyz=torch.zeros(P, 3), get_opacity=torch.ones(P, 1), get_scaling=torch.ones(P, 3),
                               get_rotation=torch.ones(P, 4), get_features=torch.zeros(P, 1, 3), active_sh_degree=0)
    cam = types.SimpleNamespace(image_height=4, image_width=4, FoVx=1.0, FoVy=1.0, world_view_transform=torch.eye(4),
                                full_proj_transform=torch.eye(4), camera_center=torch.zeros(3))
    old = GR.GaussianRasterizer
    try:
        GR.GaussianRasterizer = RefSignature
        out = GR.render(cam, pc, types.SimpleNamespace(), torch.zeros(3))
        assert out["depth_3dgs"].shape == (1, 4, 4) and made == [{}]
        GR.GaussianRasterizer = WithDepth
        GR.render(cam, pc, types.SimpleNamespace(), torch.zeros(3), depth_grad=True)
        assert made[-1] == {"depth_grad": True}
    finally:
        GR.GaussianRasterizer = old


# ---- GPU ------------------------------------------------------------------------------------------------------------

def run_gpu(cloud, cam, bg, gC=None, gD=None, gA=None, depth_grad=True, colors_precomp=None, cov3D_precomp=None,
            camera_grad=False, seed_loss_with_depth=False):
    """One forward + backward through GaussianRasterizer; loss = sum gC*colour + sum gD*depth + sum gA*alpha."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    cam_t = {}
    if camera_grad:
        cam_t = dict(viewmatrix=rs.viewmatrix.clone().requires_grad_(True),
                     projmatrix=rs.projmatrix.clone().requires_grad_(True), campos=rs.campos.clone().requires_grad_(True))
        rs = rs._replace(**cam_t)
    rast = GaussianRasterizer(rs, return_alpha=gA is not None, camera_grad=camera_grad, depth_grad=depth_grad)
    kw = dict(means3D=ct["means3D"], means2D=m2, opacities=ct["opacities"])
    leaves = dict(dmean3D=ct["means3D"], dmean2D=m2, dopacity=ct["opacities"])
    if colors_precomp is not None:
        kw["colors_precomp"] = leaves["dcolor"] = torch.from_numpy(colors_precomp).to(dev).requires_grad_(True)
    else:
        kw["shs"] = leaves["dsh"] = ct["shs"]
    if cov3D_precomp is not None:
        kw["cov3D_precomp"] = leaves["dcov3D"] = torch.from_numpy(cov3D_precomp).to(dev).requires_grad_(True)
    else:
        kw.update(scales=ct["scales"], rotations=ct["rotations"])
        leaves.update(dscale=ct["scales"], drot=ct["rotations"])
    out = rast(**kw)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    loss = 0.0
    if gC is not None:
        loss = loss + (out[0] * T(gC)).sum()
    if gD is not None:
        loss = loss + (out[2][0] * T(gD)).sum()
    if gA is not None:
        loss = loss + (out[3][0] * T(gA)).sum()
    loss.backward()
    grads = {k: (v.grad.detach().cpu().numpy() if v.grad is not None else np.zeros(tuple(v.shape), np.float32))
             for k, v in leaves.items()}
    for k, v in cam_t.items():
        grads[k] = v.grad.detach().cpu().numpy()
    return dict(out=[o.detach() if torch.is_tensor(o) else o for o in out], grads=grads)


def _check_vs_truth(got, truth, tol, skip=()):
    for k, g in got["grads"].items():
        if k in truth and k not in skip:
            want = np.asarray(truth[k])
            if np.linalg.norm(want) == 0:
                assert np.abs(g).max() == 0.0, k
                continue
            err = rel_l2(g.reshape(want.shape), want)
            assert err <= tol, (k, err)


def _small_scene(case):
    cloud, _ = synth.make_config("c3", P=20_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 192, 144, 61.0)[5]
    bg, cp, cov = (0.0, 0.0, 0.0), None, None
    if case == "deg0":
        cloud.shs = np.ascontiguousarray(cloud.shs[:, :1, :])
        cloud.sh_degree = 0
    elif case == "colors_precomp":
        cp = np.random.default_rng(3).uniform(size=(cloud.means3D.shape[0], 3)).astype(np.float32)
    elif case == "cov3D_precomp":
        f = O.forward_from(cloud, cam, render=False)
        cov = np.ascontiguousarray(f.cov3D.astype(np.float32))
        f.close()
    elif case == "background":
        bg = (0.7, 0.4, 0.9)
    return cloud, cam, bg, cp, cov


@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["depth", "colour_depth"])
@pytest.mark.parametrize("case", ["deg0", "deg3", "colors_precomp", "cov3D_precomp", "background"])
def test_small_scenes_match_fp64(case, loss):
    cloud, cam, bg, cp, cov = _small_scene(case)
    H, W = cam.image_height, cam.image_width
    rng = np.random.default_rng(21)
    gC = rng.uniform(size=(3, H, W)).astype(np.float32) if loss == "colour_depth" else None
    gD = rng.uniform(-1, 1, size=(H, W)).astype(np.float32)
    got = run_gpu(cloud, cam, bg, gC=gC, gD=gD, colors_precomp=cp, cov3D_precomp=cov)
    truth = depth_truth(cloud, cam, bg, gC=gC, gD=gD, colors_precomp=cp, cov3D_precomp=cov)
    truth["fwd"].close()
    _check_vs_truth(got, truth, 1e-4)
    assert np.linalg.norm(got["grads"]["dmean3D"]) > 0


def _gpu_depth_as_colour(cloud, cam, gD):
    """The identity on the GPU in fp32: the default path rendering colours (z, 0, 0) with background 0 and upstream
    (gD, 0, 0), z the splat records' own view depth. Returns (grads, dL/dz)."""
    from gaussianeditor_b200.rasterizer import _RasterizeGaussians, forward_state_views
    plain = run_gpu(cloud, cam, (0.0, 0.0, 0.0), gC=np.zeros((3,) + gD.shape, np.float32), depth_grad=False)
    z = forward_state_views(_RasterizeGaussians.last_state)["records"][:, 6].cpu().numpy().copy()
    z[plain["out"][1].cpu().numpy() == 0] = 0.0
    cols = np.stack([z, np.zeros_like(z), np.zeros_like(z)], 1).astype(np.float32)
    gC = np.zeros((3,) + gD.shape, np.float32)
    gC[0] = gD
    r = run_gpu(cloud, cam, (0.0, 0.0, 0.0), gC=gC, depth_grad=False, colors_precomp=cols)
    return r["grads"], r["grads"]["dcolor"][:, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["needle", "frustum_edge", "opacity_edge"])
def test_hard_scenes(scene):
    """Needle, frustum-edge and opacity-edge scenes with a colour + depth loss. Frustum- and opacity-edge: every gradient
    against the fp64 truth (1e-4). The needle's fp32 conic is too ill-conditioned for an fp64 yardstick (see
    test_parity_gpu.py::test_needle_backward_blend_weights_every_variant), so there the depth part is checked against
    the same identity evaluated by the default fp32 path on the GPU: a colour channel holding z. Only the blend's
    outputs are compared there: the needle's conic also makes the fp32 preprocess backward (dL/dmean3D, scale,
    rotation) depend on the rounding order of large cancelling terms, so adding dL/dz inside or after dL/dt.z already
    moves dL/dmean3D by ~15 %."""
    cp = None
    if scene == "needle":
        cloud, cam = synth.needle_cloud()
    elif scene == "frustum_edge":
        cloud, cam = synth.frustum_edge_cloud()
    else:
        cloud, cam = synth.opacity_edge_cloud()
    H, W = cam.image_height, cam.image_width
    rng = np.random.default_rng(5)
    gD = rng.uniform(-1, 1, size=(H, W)).astype(np.float32)
    if scene == "needle":
        only = run_gpu(cloud, cam, (0.0, 0.0, 0.0), gD=gD)["grads"]
        ident, dz = _gpu_depth_as_colour(cloud, cam, gD)
        assert np.abs(dz).max() > 0
        for k in ("dmean2D", "dopacity"):
            assert rel_l2(only[k], ident[k]) <= 1e-5, (k, rel_l2(only[k], ident[k]))
        return
    gC = rng.uniform(size=(3, H, W)).astype(np.float32)
    bg = (0.1, 0.2, 0.3)
    got = run_gpu(cloud, cam, bg, gC=gC, gD=gD, colors_precomp=cp)
    truth = depth_truth(cloud, cam, bg, gC=gC, gD=gD, colors_precomp=cp)
    truth["fwd"].close()
    _check_vs_truth(got, truth, 1e-4)


@pytest.mark.gpu
def test_full_size_config3():
    """Config 3 (1M Gaussians, 1600x1200), colour + depth loss: every gradient within 5e-5 of the fp64 truth."""
    cloud, cams = synth.make_config("c3")
    cam = cams[-1]
    H, W = cam.image_height, cam.image_width
    rng = np.random.default_rng(11)
    gC = rng.uniform(size=(3, H, W)).astype(np.float32)
    gD = rng.uniform(-0.5, 0.5, size=(H, W)).astype(np.float32)
    bg = (0.1, 0.2, 0.3)
    got = run_gpu(cloud, cam, bg, gC=gC, gD=gD)
    truth = depth_truth(cloud, cam, bg, gC=gC, gD=gD)
    truth["fwd"].close()
    _check_vs_truth(got, truth, 5e-5)


def _medium():
    cloud, _ = synth.make_config("c3", P=40_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 333, 201, 61.0)[2]     # partial last tile row and column
    rng = np.random.default_rng(23)
    H, W = cam.image_height, cam.image_width
    return cloud, cam, rng.uniform(size=(3, H, W)).astype(np.float32), rng.uniform(-1, 1, size=(H, W)).astype(np.float32)


@pytest.mark.gpu
def test_default_drops_depth_and_opt_in_fast_path():
    """depth_grad=False: a depth term changes nothing. depth_grad=True with a colour-only loss takes the ordinary
    backward, and a depth-only loss works. Two backward passes are not bit-identical even on the same path (the
    blending backward sums with float atomics; two runs of one build differ by ~1e-7 relative L2 at config 3), so
    "the same" is: within 1e-6, where the depth term would move them by O(1)."""
    cloud, cam, gC, gD = _medium()
    bg = (0.2, 0.3, 0.4)
    base = run_gpu(cloud, cam, bg, gC=gC, depth_grad=False)["grads"]
    with_d = run_gpu(cloud, cam, bg, gC=gC, gD=gD, depth_grad=False)["grads"]
    fast = run_gpu(cloud, cam, bg, gC=gC, depth_grad=True)["grads"]
    only = run_gpu(cloud, cam, bg, gD=gD)["grads"]
    for k in base:
        assert rel_l2(with_d[k], base[k]) <= 1e-6, k
        assert rel_l2(fast[k], base[k]) <= 1e-6, k
    assert rel_l2(run_gpu(cloud, cam, bg, gC=gC, gD=gD)["grads"]["dmean3D"], base["dmean3D"]) > 1e-2
    assert np.linalg.norm(only["dmean3D"]) > 0 and np.isfinite(only["dmean3D"]).all()
    assert not only["dsh"].any()     # the depth does not depend on the colour


@pytest.mark.gpu
def test_linearity():
    cloud, cam, gC, gD = _medium()
    bg = (0.2, 0.3, 0.4)
    both = run_gpu(cloud, cam, bg, gC=gC, gD=gD)["grads"]
    c = run_gpu(cloud, cam, bg, gC=gC)["grads"]
    d = run_gpu(cloud, cam, bg, gD=gD)["grads"]
    for k in both:
        assert rel_l2(both[k], c[k].astype(np.float64) + d[k]) <= 1e-6, (k, rel_l2(both[k], c[k].astype(np.float64) + d[k]))


@pytest.mark.gpu
def test_with_alpha_matches_fp64():
    cloud, cam, gC, gD = _medium()
    gA = np.random.default_rng(29).uniform(-1, 1, size=gD.shape).astype(np.float32)
    bg = (0.2, 0.3, 0.4)
    got = run_gpu(cloud, cam, bg, gC=gC, gD=gD, gA=gA)
    assert len(got["out"]) == 4
    truth = depth_truth(cloud, cam, bg, gC=gC, gD=gD, gA=gA)
    truth["fwd"].close()
    _check_vs_truth(got, truth, 1e-4)


@pytest.mark.gpu
def test_with_camera_gradients():
    """dL/dviewmatrix = camera_grads_formulas on the fp64 upstream sums + sum dL/dz (x, y, z, 1) on entries 2, 6, 10, 14
    (1e-3), and central finite differences of the fp64 oracle's colour + depth loss (6 %, the bound and the reasoning
    of test_camera_gradients_match_the_fp64_oracle_chain_and_finite_differences)."""
    from test_camera_grad_math import camera_grads_formulas
    cloud, _ = synth.make_config("c3", P=4000)
    cloud.shs = np.ascontiguousarray(cloud.shs[:, :4, :])
    cloud.sh_degree = 1
    cam = synth.ring_cameras(8, 4.5, 15.0, 96, 64, 61.0)[3]
    H, W = cam.image_height, cam.image_width
    bg = (0.2, 0.1, 0.3)
    rng = np.random.default_rng(31)
    gC = rng.uniform(0.5, 1.5, size=(3, H, W)).astype(np.float32)
    gD = rng.uniform(0.1, 0.3, size=(H, W)).astype(np.float32)
    got = run_gpu(cloud, cam, bg, gC=gC, gD=gD, camera_grad=True)["grads"]
    assert np.all(got["viewmatrix"][:, 3] == 0)

    g = depth_truth(cloud, cam, bg, gC=gC, gD=gD)
    f = g["fwd"]
    vis = f.radii > 0
    hx, hy = W / (2 * cam.tanfovx), H / (2 * cam.tanfovy)
    g_conic = np.stack([g["dconic"][vis, 0, 0], g["dconic"][vis, 0, 1], g["dconic"][vis, 1, 1]], 1)
    g_col = g["dcolor"][vis] * (1.0 - f.clamped[vis].astype(np.float64))
    means = cloud.means3D[vis].astype(np.float64)
    dv, dp, dc = camera_grads_formulas(cam.viewmatrix.astype(np.float64), cam.projmatrix.astype(np.float64),
                                       cam.campos.astype(np.float64), means, f.cov3D[vis].astype(np.float64),
                                       cloud.shs[vis].astype(np.float64), g["dmean2D"][vis, :2], g_conic, g_col, hx, hy)
    mj = np.concatenate([means, np.ones((means.shape[0], 1))], 1)
    dv = dv.copy()
    dv[:, 2] += (g["ddepth"][vis][:, None] * mj).sum(0)     # dview[2 + 4j], row-major [j][2]
    f.close()
    for name, want in (("viewmatrix", dv), ("projmatrix", dp), ("campos", dc)):
        assert rel_l2(got[name], want) <= 1e-3, (name, rel_l2(got[name], want))

    def loss(view):
        ff = O.forward_from(cloud, cam, bg, f32=False, viewmatrix=view)
        v = float((ff.color * gC).sum() + (ff.depth[0] * gD).sum())
        ff.close()
        return v
    h = np.float32(2.0 ** -11)
    arr = cam.viewmatrix.astype(np.float32)
    fd = np.zeros(arr.shape, np.float64)
    for idx in np.ndindex(arr.shape):
        if idx[1] == 3:
            continue
        ap, am = arr.copy(), arr.copy()
        ap[idx] += h; am[idx] -= h
        fd[idx] = (loss(ap) - loss(am)) / float(ap[idx] - am[idx])
    assert rel_l2(got["viewmatrix"], fd) <= 6e-2, (rel_l2(got["viewmatrix"], fd), got["viewmatrix"], fd)


@pytest.mark.gpu
def test_fused_activations():
    """forward_raw with depth_grad=True against the PyTorch-activated path with depth_grad=True, with the bounds of
    test_fused_activations_match_pytorch_prologue."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    from test_parity_gpu import _raw_params
    dev = torch.device("cuda")
    cloud, _ = synth.make_config("c3", P=60013)
    cam = synth.ring_cameras(8, 4.5, 15.0, 640, 400, 61.0)[1]
    rs = settings_from(cam, (0.3, 0.1, 0.2), 3, dev)
    rng = np.random.default_rng(5)
    dL = torch.from_numpy(rng.uniform(size=(3, 400, 640)).astype(np.float32)).to(dev)
    dD = torch.from_numpy(rng.uniform(-1, 1, size=(400, 640)).astype(np.float32)).to(dev)
    rast = GaussianRasterizer(rs, depth_grad=True)
    a = _raw_params(cloud, dev)
    m2a = torch.zeros_like(a["xyz"], requires_grad=True)
    col_a, rad_a, dep_a = rast(means3D=a["xyz"], means2D=m2a, opacities=torch.sigmoid(a["opacity"]),
                               shs=torch.cat((a["features_dc"], a["features_rest"]), dim=1),
                               scales=torch.exp(a["scaling"]), rotations=torch.nn.functional.normalize(a["rotation"]))
    ((col_a * dL).sum() + (dep_a[0] * dD).sum()).backward()
    b = _raw_params(cloud, dev)
    m2b = torch.zeros_like(b["xyz"], requires_grad=True)
    col_b, rad_b, dep_b = rast.forward_raw(means3D=b["xyz"], means2D=m2b, opacity_logits=b["opacity"],
                                           features_dc=b["features_dc"], features_rest=b["features_rest"],
                                           log_scales=b["scaling"], raw_rotations=b["rotation"])
    ((col_b * dL).sum() + (dep_b[0] * dD).sum()).backward()
    assert float((rad_a != rad_b).float().mean()) <= 1e-4
    same = rad_a == rad_b
    for k in a:
        ga, gb = a[k].grad, b[k].grad
        assert gb is not None and torch.isfinite(gb).all(), k
        assert rel_l2(gb[same].cpu().numpy(), ga[same].cpu().numpy()) <= 1e-4, k
    assert rel_l2(m2b.grad[same].cpu().numpy(), m2a.grad[same].cpu().numpy()) <= 1e-4
    # depth alone on the fused path
    c = _raw_params(cloud, dev)
    _, _, dep_c = rast.forward_raw(means3D=c["xyz"], means2D=torch.zeros_like(c["xyz"]), opacity_logits=c["opacity"],
                                   features_dc=c["features_dc"], features_rest=c["features_rest"],
                                   log_scales=c["scaling"], raw_rotations=c["rotation"])
    (dep_c[0] * dD).sum().backward()
    assert float(c["xyz"].grad.abs().sum()) > 0 and float(c["features_dc"].grad.abs().sum()) == 0.0


@pytest.mark.gpu
def test_edge_cases():
    """P = 0, every Gaussian culled, and a partial last tile row and column (333x201, in _medium), with depth_grad."""
    cam = synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 64, 48, fovy_deg=50.0)
    empty = synth.Cloud(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros((0, 4), np.float32),
                        np.zeros((0, 1), np.float32), np.zeros((0, 1, 3), np.float32), 0)
    gD = np.ones((48, 64), np.float32)
    r = run_gpu(empty, cam, (0.3, 0.2, 0.1), gC=np.ones((3, 48, 64), np.float32), gD=gD, camera_grad=True,
                colors_precomp=np.zeros((0, 3), np.float32))
    assert all(v.size == 0 for k, v in r["grads"].items() if k.startswith("d"))
    assert not r["grads"]["viewmatrix"].any()
    c, _ = synth.make_config("c1", P=500)
    c.means3D[:, 2] = -10.0
    r = run_gpu(c, cam, (0.3, 0.2, 0.1), gD=gD)
    assert int((r["out"][1] > 0).sum()) == 0
    for k, g in r["grads"].items():
        assert not g.any(), k
    cloud, cam2, gC, gD2 = _medium()
    got = run_gpu(cloud, cam2, (0.0, 0.0, 0.0), gC=gC, gD=gD2)
    truth = depth_truth(cloud, cam2, (0.0, 0.0, 0.0), gC=gC, gD=gD2)
    truth["fwd"].close()
    _check_vs_truth(got, truth, 1e-4)
