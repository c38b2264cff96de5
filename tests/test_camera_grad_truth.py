"""Camera-pose gradients (``GaussianRasterizer(..., camera_grad=True)``) against an fp64 autograd truth.

The truth (``camera_truth``) restates in torch float64 the per-Gaussian FORWARD map

    (viewmatrix, projmatrix, campos)  ->  (mean2D in NDC, conic, SH colour, view depth z)

and lets autograd differentiate  sum_i  g_mean2D . mean2D + g_conic . conic + g_colour . rgb + g_z . z  for fixed
upstream gradients g: what the blend backward hands to the preprocess backward. The upstream comes from the fp64 CPU
oracle of the same scene and loss (``test_depth_grad.depth_truth``: colour, depth and alpha terms), never from the GPU
forward's own state. The map follows the forward as the kernels compute it:

* mean2D = p_hom.xy / (p_hom.w + 1e-7); the focal lengths h_x = W / (2 tan_fovx), h_y likewise, rounded to float32
  as the kernel rounds them (``focal="f64"`` takes the oracle's unrounded ones); the 2-D covariance gets the +0.3
  dilation before it is inverted to the conic.
* The SH colour at degrees 0-3, the active degree at most the allocated one, plus 0.5; a channel the oracle reports
  ``clamped`` (colour < 0) passes no gradient. ``colors_precomp`` skips the SH entirely: campos then gets exactly 0, and
  so it does at degree 0. SH constants are the float32 ones of the kernels and the oracle.
* The covariance comes from scale (times ``scale_modifier``) and rotation, or from ``cov3D_precomp``; it does not depend
  on the camera, and the truth checks its own restatement against the oracle's.
* Under ``depth_grad`` the view depth z = t.z (not clamped) adds g_z to the derivative of t.z.

Semantics of the camera gradient at the Jacobian clamp. The forward clamps t.x / t.z to +-1.3 tan_fovx (and y alike)
before it builds the projection Jacobian J. The camera gradient follows the reference's convention for the mean
gradient, and so must ``dL/dmeans3D`` for parity: where |t.x / t.z| > limx, dL/dt.x is zero and the clamped t.x is a
constant in the t.z derivative of J02. As a formula:

    tx_c = where(|tx / tz| > limx,  (clamp(tx / tz, -limx, limx) * tz).detach(),  tx)        (and likewise for y)

This is not the derivative of the clamped map (which would let tx_c = limx * tz follow t.z); ``test_clamp_convention``
writes the convention out and shows that the two differ. Because the camera gradient and dL/dmeans3D use one dL/dt,
moving the world by a translation leaves the loss unchanged under either convention, and the translation identity
holds exactly in fp64 (``test_translation_identity_fp64``).

Two conventions of the backward are modelled as scalings of the upstream, not as part of the forward:
* the blend backward hands over HALF of dL/d(conic b) (see test_camera_grad_math.py), so the truth takes 2 x the
  oracle's dconic[0, 1];
* the preprocess backward divides by denom^2 + 1e-7 instead of denom^2 (denom = a c - b^2 of the dilated 2-D
  covariance), a relative change of up to ~1e-5 for pixel-sized splats; the truth scales each Gaussian's conic upstream
  by denom^2 / (denom^2 + 1e-7), which is what the kernels and the oracle compute.

The truth also returns, for every output entry e, B_e = sum_i |c_{i,e}|: the sum of the absolute per-Gaussian
contributions (each Gaussian gets its own copy of the camera arrays as an autograd leaf). A float32 sum of those
contributions is off by a few ulp of B_e, not of the (possibly much smaller) total, so every GPU bound is element-wise
|got_e - truth_e| <= TAU * B_e, plus a relative L2 bound RHO per array, plus exact zeros where B_e = 0 (view column 3
and proj column 2 in the [4, 4] indexing of the returned gradients, which the forward never reads).

TAU, RHO and TAU_ID are set from measurements on an H100 80GB HBM3 (700 W power limit), with headroom of 3.5x or more.
Over every GPU case below, the 1M-Gaussian config 3 included, the largest |got - truth| / B_e was 4.1e-6 (5.6e-5 on the
frustum-edge scene, whose near-cut rows and zero scale axes make the per-Gaussian fp32 terms cancel more, hence
TAU_EDGE). The largest relative L2 was 4.5e-6 for viewmatrix, 1.3e-6 for campos and 1.1e-4 for projmatrix. The
projection's gradient is a sum of terms of both signs (dL/dmean2D . mean) whose total is ~1e-2 of B, so its relative
L2 measures that cancellation, not the kernel; the element-wise bound is the tight check for it. The translation
identity on the GPU outputs held to 3.2e-8 of its summed magnitudes.

Rows whose radii differ between the GPU (fp32, contracted) and the fp64 oracle would make the two sums incomparable;
``_matched`` drops them from the cloud before the comparison and asserts the radii are then identical.

Through the Python API a misaligned SH tensor is copied to aligned storage (``rasterizer._f32c``), so the SH row is
always read with the bulk copy at M = 4 and 16; the plain (non-bulk) camera kernels are reached through M = 1 and 9 and
``colors_precomp``, all covered below, each with and without ``depth_grad``.
"""
import numpy as np
import pytest
import torch

from gaussianeditor_b200 import synth
from oracle import cpu_oracle as O
from test_camera_grad_math import camera_grads_formulas
from test_depth_grad import depth_truth
from util import cloud_tensors, rel_l2, settings_from

f32 = lambda x: float(np.float32(x))
DILATION, EPS_W, EPS_DEN = f32(0.3), f32(1e-7), f32(1e-7)
SH_C0, SH_C1 = f32(0.28209479177387814), f32(0.4886025119029199)
SH_C2 = [f32(c) for c in (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                          0.5462742152960396)]
SH_C3 = [f32(c) for c in (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
                          -0.4570457994644658, 1.445305721320277, -0.5900435899266435)]
CAM = ("viewmatrix", "projmatrix", "campos")
NEVER_READ = dict(viewmatrix=(slice(None), 3), projmatrix=(slice(None), 2))   # [4, 4] indexing

TAU = 1.5e-5        # element-wise, in units of B_e
TAU_EDGE = 2e-4   # the same on synth.frustum_edge_cloud (view depths at the 0.2 near cut, zero scale axes)
RHO = dict(viewmatrix=2e-5, projmatrix=5e-4, campos=1e-5)   # relative L2 per array
RHO_POSE = 2e-4   # relative L2 of pose.grad (dominated by the projection's share)
TAU_ID = 2e-7     # translation identity on the GPU outputs, in units of the summed magnitudes of its terms


# ---- the fp64 truth -------------------------------------------------------------------------------------------------

def _focal(cam, focal="f32"):
    """(h_x, h_y, limx, limy) as the kernel (float32) or the fp64 oracle computes them."""
    if focal == "f32":
        two = np.float32(2.0)
        hx = np.float32(cam.image_width) / (two * np.float32(cam.tanfovx))
        hy = np.float32(cam.image_height) / (two * np.float32(cam.tanfovy))
        return float(hx), float(hy), float(np.float32(1.3) * np.float32(cam.tanfovx)), \
            float(np.float32(1.3) * np.float32(cam.tanfovy))
    tx, ty = float(np.float32(cam.tanfovx)), float(np.float32(cam.tanfovy))
    return cam.image_width / (2.0 * tx), cam.image_height / (2.0 * ty), f32(1.3) * tx, f32(1.3) * ty


def _sh_basis(D, x, y, z):
    b = [torch.full_like(x, SH_C0)]
    if D > 0:
        b += [-SH_C1 * y, SH_C1 * z, -SH_C1 * x]
    if D > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [SH_C2[0] * xy, SH_C2[1] * yz, SH_C2[2] * (2 * zz - xx - yy), SH_C2[3] * xz, SH_C2[4] * (xx - yy)]
    if D > 2:
        b += [SH_C3[0] * y * (3 * xx - yy), SH_C3[1] * xy * z, SH_C3[2] * y * (4 * zz - xx - yy),
              SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy), SH_C3[4] * x * (4 * zz - xx - yy), SH_C3[5] * z * (xx - yy),
              SH_C3[6] * x * (xx - 3 * yy)]
    return torch.stack(b, 1)


def cov3d_of(scales, rotations, scale_modifier=1.0):
    """fp64 3-D covariance (xx, xy, xz, yy, yz, zz) of scale * modifier and the (unnormalised) quaternion r, x, y, z."""
    s = np.asarray(scales, np.float64) * float(np.float32(scale_modifier))
    r, x, y, z = np.asarray(rotations, np.float64).T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], 1),
                  np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], 1),
                  np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1)], 1)
    S = np.einsum("pij,pj,pkj->pik", R, s * s, R)
    return np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)


def _map(v, pm, cp, sc, detach_clamp=True):
    """The forward map on per-row (or shared) camera arrays v [N|1, 16], pm [N|1, 16], cp [N|1, 3]."""
    means = sc["means"]
    x, y, z = means[:, 0], means[:, 1], means[:, 2]
    tx = v[:, 0] * x + v[:, 4] * y + v[:, 8] * z + v[:, 12]
    ty = v[:, 1] * x + v[:, 5] * y + v[:, 9] * z + v[:, 13]
    tz = v[:, 2] * x + v[:, 6] * y + v[:, 10] * z + v[:, 14]
    hw = pm[:, 3] * x + pm[:, 7] * y + pm[:, 11] * z + pm[:, 15]
    m_w = 1.0 / (hw + EPS_W)
    px = (pm[:, 0] * x + pm[:, 4] * y + pm[:, 8] * z + pm[:, 12]) * m_w
    py = (pm[:, 1] * x + pm[:, 5] * y + pm[:, 9] * z + pm[:, 13]) * m_w
    hx, hy, limx, limy = sc["focal"]

    def clamp(t, lim):
        r = t / tz
        c = r.clamp(-lim, lim) * tz
        return torch.where(r.abs() > lim, c.detach() if detach_clamp else c, t)
    txc, tyc = clamp(tx, limx), clamp(ty, limy)
    J00, J02, J11, J12 = hx / tz, -(hx * txc) / (tz * tz), hy / tz, -(hy * tyc) / (tz * tz)
    W0 = torch.stack([v[:, 0], v[:, 4], v[:, 8]], 1)
    W1 = torch.stack([v[:, 1], v[:, 5], v[:, 9]], 1)
    W2 = torch.stack([v[:, 2], v[:, 6], v[:, 10]], 1)
    T0 = W0 * J00[:, None] + W2 * J02[:, None]
    T1 = W1 * J11[:, None] + W2 * J12[:, None]
    V = sc["V"]
    a = torch.einsum("pi,pij,pj->p", T0, V, T0) + DILATION
    b = torch.einsum("pi,pij,pj->p", T0, V, T1)
    c = torch.einsum("pi,pij,pj->p", T1, V, T1) + DILATION
    det = a * c - b * b
    out = dict(px=px, py=py, A=c / det, B=-b / det, C=a / det, z=tz, det=det, clamped_xy=(
        ((tx / tz).abs() > limx) | ((ty / tz).abs() > limy)))
    if sc["sh"] is not None:
        d = means - cp
        d = d / d.norm(dim=1, keepdim=True)
        basis = _sh_basis(sc["D"], d[:, 0], d[:, 1], d[:, 2])
        rgb = torch.einsum("pk,pkc->pc", basis, sc["sh"][:, :basis.shape[1]]) + 0.5
        out["rgb"] = torch.where(sc["rgb_clamped"], torch.zeros_like(rgb), rgb)
    return out


def _proxy(v, pm, cp, sc, up, detach_clamp=True, per_row=False):
    o = _map(v, pm, cp, sc, detach_clamp)
    s = up["m2"][:, 0] * o["px"] + up["m2"][:, 1] * o["py"] + up["con"][:, 0] * o["A"] + up["con"][:, 1] * o["B"] \
        + up["con"][:, 2] * o["C"] + up["z"] * o["z"]
    if "rgb" in o:
        s = s + (up["col"] * o["rgb"]).sum(1)
    return s if per_row else s.sum()


def make_scene(cam, means, sh, D, cov3d, rgb_clamped=None, focal="f32"):
    t = lambda a: torch.as_tensor(np.asarray(a, np.float64))
    c3 = np.asarray(cov3d, np.float64)
    V = np.stack([np.stack([c3[:, 0], c3[:, 1], c3[:, 2]], 1), np.stack([c3[:, 1], c3[:, 3], c3[:, 4]], 1),
                  np.stack([c3[:, 2], c3[:, 4], c3[:, 5]], 1)], 1)
    N = means.shape[0]
    return dict(means=t(means), V=t(V), D=D, sh=None if sh is None else t(sh), focal=_focal(cam, focal),
                rgb_clamped=torch.zeros(N, 3, dtype=torch.bool) if rgb_clamped is None else torch.as_tensor(rgb_clamped),
                cam=[t(np.asarray(a, np.float32)) for a in (cam.viewmatrix.reshape(-1), cam.projmatrix.reshape(-1),
                                                          cam.campos)])


def make_upstream(sc, g_m2, g_con_oracle, g_col, g_z, eps_den=True):
    """Upstream in the truth's terms: dL/d(A, B, C) from the blend backward's (A, B/2, C), each Gaussian's row scaled
    by denom^2 / (denom^2 + 1e-7) when eps_den (the preprocess backward's epsilon)."""
    t = lambda a: torch.as_tensor(np.asarray(a, np.float64))
    con = t(g_con_oracle) * torch.tensor([1.0, 2.0, 1.0], dtype=torch.float64)
    if eps_den:
        with torch.no_grad():
            den = _map(*(a[None] for a in sc["cam"]), sc)["det"]
        con = con * (den * den / (den * den + EPS_DEN))[:, None]
    return dict(m2=t(g_m2), con=con, col=t(g_col), z=t(g_z))


def truth_rows(sc, up, detach_clamp=True):
    """autograd with a per-Gaussian copy of each camera array -> (sum over rows, sum of |rows|, rows) per array."""
    N = sc["means"].shape[0]
    leaves = [a[None].expand(N, -1).clone().requires_grad_(True) for a in sc["cam"]]
    _proxy(*leaves, sc, up, detach_clamp).backward()
    shapes = dict(viewmatrix=(4, 4), projmatrix=(4, 4), campos=(3,))
    truth, B, rows = {}, {}, {}
    for name, leaf in zip(CAM, leaves):
        g = np.zeros(tuple(leaf.shape)) if leaf.grad is None else leaf.grad.numpy()   # None: nothing reads it
        truth[name], B[name], rows[name] = g.sum(0).reshape(shapes[name]), np.abs(g).sum(0).reshape(shapes[name]), g
    return truth, B, rows


def camera_truth(cloud, cam, bg, gC=None, gD=None, gA=None, colors_precomp=None, cov3D_precomp=None,
                 scale_modifier=1.0, focal="f32"):
    """fp64 camera gradients of  sum gC*colour + sum gD*depth + sum gA*alpha  -> dict with ``truth`` and ``B`` (per array),
    the oracle's gradient dict ``g`` (dmean3D included) and the fp64 forward ``f`` (closed)."""
    g = depth_truth(cloud, cam, bg, gC=gC, gD=gD, gA=gA, colors_precomp=colors_precomp, cov3D_precomp=cov3D_precomp,
                    scale_modifier=scale_modifier)
    f = g.pop("fwd")
    f.close()
    vis = f.radii > 0
    cov = cov3D_precomp.astype(np.float64) if cov3D_precomp is not None else \
        cov3d_of(cloud.scales, cloud.rotations, scale_modifier)
    assert np.abs(cov[vis] - f.cov3D[vis]).max() <= 1e-12 * max(np.abs(f.cov3D[vis]).max(), 1e-30)
    sh = None if colors_precomp is not None else cloud.shs[vis]
    sc = make_scene(cam, cloud.means3D[vis], sh, cloud.sh_degree, cov[vis], f.clamped[vis].astype(bool), focal)
    con = np.stack([g["dconic"][vis, 0, 0], g["dconic"][vis, 0, 1], g["dconic"][vis, 1, 1]], 1)
    up = make_upstream(sc, g["dmean2D"][vis, :2], con, g["dcolor"][vis], g["ddepth"][vis])
    truth, B, _ = truth_rows(sc, up)
    clamped_xy = _map(*(a[None] for a in sc["cam"]), sc)["clamped_xy"].numpy()
    return dict(truth=truth, B=B, g=g, vis=vis, clamped_xy=clamped_xy, rgb_clamped=f.clamped[vis])


def translation_identity(dmean3D, cam_grads, view, proj):
    """sum_i dmean3D_i + dcampos - R_view^T dview[3, :3] - P_R^T dproj[3, :] (the derivative of the loss under a shift of
    the world, which is 0) and the summed magnitudes of its terms."""
    V, Pm = np.asarray(view, np.float64).reshape(4, 4), np.asarray(proj, np.float64).reshape(4, 4)
    dv, dp, dc = (np.asarray(cam_grads[k], np.float64) for k in CAM)
    dv, dp = dv.reshape(4, 4), dp.reshape(4, 4)
    # t_k = sum_j V[j, k] m_j + V[3, k]: shifting the world by delta moves V[3, k] by -sum_j V[j, k] delta_j
    tv = V[:3, :3] @ dv[3, :3]
    tp = Pm[:3, :] @ dp[3, :]
    dm = np.asarray(dmean3D, np.float64)
    s = dm.sum(0) + dc - tv - tp
    mag = np.abs(dm).sum(0) + np.abs(dc) + np.abs(V[:3, :3]) @ np.abs(dv[3, :3]) + np.abs(Pm[:3, :]) @ np.abs(dp[3, :])
    return s, mag


# ---- CPU: the truth itself --------------------------------------------------------------------------------------------

def _random_scene(deg, M=None, P=40, seed=0, spread=0.6):
    rng = np.random.default_rng(seed)
    cam = synth.ring_cameras(8, 4.5, 15.0, 96, 64, 61.0)[3]
    M = (deg + 1) ** 2 if M is None else M
    means = rng.normal(0, spread, (P, 3))
    Lm = rng.normal(0, 0.05, (P, 3, 3))
    S = np.einsum("pij,pkj->pik", Lm, Lm) + 1e-4 * np.eye(3)
    cov3d = np.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)
    sh = rng.normal(0, 0.5, (P, M, 3))
    ups = rng.normal(size=(P, 2)), rng.normal(size=(P, 3)), rng.normal(size=(P, 3)), rng.normal(size=P)
    return cam, means, cov3d, sh, ups


def test_truth_equals_the_kernel_formulas_on_unclamped_rows(monkeypatch):
    """Degree 1, no Jacobian clamp, no depth term, conic epsilon off: the autograd truth equals camera_grads_formulas
    (the line-by-line restatement of the kernel, itself tied to autograd in test_camera_grad_math.py) to 1e-9. The
    formulas write the constants 0.3, 1e-7 and C0, C1 in decimal; the truth takes them so for this comparison."""
    import test_camera_grad_truth as me
    for k, v in dict(DILATION=0.3, EPS_W=1e-7, SH_C0=0.28209479177387814, SH_C1=0.4886025119029199).items():
        monkeypatch.setattr(me, k, v)
    cam, means, cov3d, sh, (g_m2, g_con, g_col, _) = _random_scene(1)
    sc = make_scene(cam, means, sh, 1, cov3d, focal="f64")
    assert not _map(*(a[None] for a in sc["cam"]), sc)["clamped_xy"].any()
    up = make_upstream(sc, g_m2, g_con, g_col, np.zeros(len(means)), eps_den=False)
    truth, B, _ = truth_rows(sc, up)
    hx, hy, _, _ = _focal(cam, "f64")
    view, proj, cpos = (np.asarray(a, np.float32).astype(np.float64) for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    dv, dp, dc = camera_grads_formulas(view, proj, cpos, means, cov3d, sh, g_m2, g_con, g_col, hx, hy)
    for name, want in zip(CAM, (dv, dp, dc)):
        assert np.linalg.norm(want) > 0
        assert rel_l2(truth[name], want) <= 1e-9, (name, rel_l2(truth[name], want))
        assert np.all(B[name] >= np.abs(truth[name]))
    for name, idx in NEVER_READ.items():
        assert not truth[name][idx].any() and not B[name][idx].any()


def _reference_dt(sc, up):
    """dL/dt per Gaussian as the reference writes it (backward.cu:244-253 and the kernel): dL/dt.x zeroed where
    |t.x / t.z| > limx, and 2 h_x t.x' / t.z^3 dL/dJ02 in dL/dt.z with the CLAMPED t.x' (y alike). numpy float64."""
    v, pm, _ = (a.numpy() for a in sc["cam"])
    m = sc["means"].numpy()
    hx, hy, limx, limy = sc["focal"]
    t = np.stack([m @ v[[0, 4, 8]] + v[12], m @ v[[1, 5, 9]] + v[13], m @ v[[2, 6, 10]] + v[14]], 1)
    rx, ry = t[:, 0] / t[:, 2], t[:, 1] / t[:, 2]
    xm, ym = (np.abs(rx) <= limx).astype(float), (np.abs(ry) <= limy).astype(float)
    tx, ty, tz = np.clip(rx, -limx, limx) * t[:, 2], np.clip(ry, -limy, limy) * t[:, 2], t[:, 2]
    J00, J02, J11, J12 = hx / tz, -hx * tx / tz ** 2, hy / tz, -hy * ty / tz ** 2
    W = np.stack([v[[0, 4, 8]], v[[1, 5, 9]], v[[2, 6, 10]]])
    T0 = W[0][None] * J00[:, None] + W[2][None] * J02[:, None]
    T1 = W[1][None] * J11[:, None] + W[2][None] * J12[:, None]
    V = sc["V"].numpy()
    a = np.einsum("pi,pij,pj->p", T0, V, T0) + DILATION
    b = np.einsum("pi,pij,pj->p", T0, V, T1)
    c = np.einsum("pi,pij,pj->p", T1, V, T1) + DILATION
    con = up["con"].numpy()
    gA, gB, gC = con[:, 0], con[:, 1] / 2, con[:, 2]
    den = a * c - b * b
    d2 = 1.0 / den ** 2
    dA = d2 * (-c * c * gA + 2 * b * c * gB + (den - a * c) * gC)
    dC = d2 * (-a * a * gC + 2 * a * b * gB + (den - a * c) * gA)
    dB = d2 * 2 * (b * c * gA - (den + 2 * b * b) * gB + a * b * gC)
    u0, u1 = np.einsum("pij,pj->pi", V, T0), np.einsum("pij,pj->pi", V, T1)
    dT0 = 2 * u0 * dA[:, None] + u1 * dB[:, None]
    dT1 = 2 * u1 * dC[:, None] + u0 * dB[:, None]
    dJ00, dJ02, dJ11, dJ12 = dT0 @ W[0], dT0 @ W[2], dT1 @ W[1], dT1 @ W[2]
    dtx = xm * -hx * dJ02 / tz ** 2
    dty = ym * -hy * dJ12 / tz ** 2
    dtz = -hx * dJ00 / tz ** 2 - hy * dJ11 / tz ** 2 + 2 * hx * tx * dJ02 / tz ** 3 + 2 * hy * ty * dJ12 / tz ** 3
    up_z = up["z"].numpy()
    return np.stack([dtx, dty, dtz + up_z], 1), (xm == 0) | (ym == 0)


def test_clamp_convention():
    """On clamped rows the truth's dL/dt (a Gaussian's own gradient of view[12..14], since t = ... + view[12 + k])
    equals the reference convention written out (1e-12), and differs from the derivative of the clamped map without
    the detach, so a change of convention would be noticed. The scene spreads the centres to |x / z| up to ~2 limx."""
    cam, means, cov3d, sh, (g_m2, g_con, g_col, g_z) = _random_scene(1, P=400, seed=3, spread=2.5)
    tz = means @ cam.viewmatrix.astype(np.float64)[:3, 2] + float(cam.viewmatrix[3, 2])
    keep = tz > 0.5
    sc = make_scene(cam, means[keep], sh[keep], 1, cov3d[keep], focal="f64")
    up = make_upstream(sc, g_m2[keep], g_con[keep], g_col[keep], g_z[keep], eps_den=False)
    _, _, rows = truth_rows(sc, up)
    got = rows["viewmatrix"][:, 12:15]
    want, clamped = _reference_dt(sc, up)
    assert clamped.sum() >= 20 and (~clamped).sum() >= 20, clamped.sum()
    scale = np.abs(want).max(1)
    assert np.all(np.abs(got - want).max(1) <= 1e-12 * np.maximum(scale, 1e-30)), np.abs(got - want).max()
    _, _, rows_nd = truth_rows(sc, up, detach_clamp=False)
    nd = rows_nd["viewmatrix"][:, 12:15]
    assert np.all(np.abs(nd[~clamped] - got[~clamped]).max(1) <= 1e-14 * np.abs(got[~clamped]).max(1))
    diff = np.abs(nd[clamped] - got[clamped]).max(1) / np.abs(got[clamped]).max(1)
    assert np.median(diff) > 1e-2, np.median(diff)


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_finite_differences_of_the_proxy(deg):
    """Central differences of the fixed-upstream proxy (smooth, unlike the rendered image) in fp64 agree with the truth
    to 1e-7 relative L2 for all three arrays, at every SH degree, on a scene without clamped rows."""
    cam, means, cov3d, sh, (g_m2, g_con, g_col, g_z) = _random_scene(deg, seed=10 + deg)
    sc = make_scene(cam, means, sh, deg, cov3d, focal="f64")
    assert not _map(*(a[None] for a in sc["cam"]), sc)["clamped_xy"].any()
    up = make_upstream(sc, g_m2, g_con, g_col, g_z)
    truth, _, _ = truth_rows(sc, up)
    base = [a.clone() for a in sc["cam"]]
    h = 1e-4
    for i, name in enumerate(CAM):
        fd = np.zeros(base[i].numel())
        for e in range(base[i].numel()):
            f = {}
            for k in (-2, -1, 1, 2):
                arrs = [a.clone() for a in base]
                arrs[i][e] += k * h
                f[k] = _proxy(*(a[None] for a in arrs), sc, up, per_row=True)
            # fourth-order central stencil, differenced per Gaussian before the sum
            fd[e] = float(((f[-2] - f[2]) + 8.0 * (f[1] - f[-1])).sum()) / (12.0 * h)
        want = truth[name].reshape(-1)
        if name == "campos" and deg == 0:
            assert not want.any() and np.abs(fd).max() <= 1e-9
            continue
        assert rel_l2(fd, want) <= 1e-7, (name, rel_l2(fd, want))


@pytest.mark.parametrize("case", ["deg1", "deg3_clamped", "depth_alpha"])
def test_translation_identity_fp64(case):
    """Moving the world by delta (means and campos by delta, the view's translation by -R_view delta, the projection's
    by -P_R delta) leaves the image unchanged, so sum_i dmean3D_i + dcampos minus the two translation terms is 0. With
    the ORACLE's own dmean3D and the truth's camera gradients this holds to 1e-10 of the summed magnitudes, clamped rows
    included: the camera truth and the oracle's mean gradient share one convention."""
    cloud, cam, bg, gC, gD, gA = _cpu_scene(case)
    r = camera_truth(cloud, cam, bg, gC=gC, gD=gD, gA=gA, focal="f64")
    if case == "deg3_clamped":
        assert r["clamped_xy"].sum() >= 10 and r["rgb_clamped"].any()
    s, mag = translation_identity(r["g"]["dmean3D"], r["truth"], cam.viewmatrix, cam.projmatrix)
    assert np.all(np.abs(s) <= 1e-10 * mag), (s, mag)
    assert np.linalg.norm(r["truth"]["campos"]) > 0


def _cpu_scene(case):
    H, W = 48, 64
    rng = np.random.default_rng(41)
    gC = rng.uniform(-0.5, 1.5, size=(3, H, W)).astype(np.float32)
    gD = gA = None
    if case == "deg3_clamped":
        cloud, cam = _clamp_heavy(n=1500)
        cloud.shs[:, 0, 0] -= np.float32(0.4 / 0.28209479177387814)
        gC = rng.uniform(-0.5, 1.5, size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    else:
        cloud, _ = synth.make_config("c3", P=2000)
        if case == "deg1":
            cloud.shs = np.ascontiguousarray(cloud.shs[:, :4, :])
            cloud.sh_degree = 1
        cam = synth.look_at_camera((0, 0.5, -4.0), (0, 0, 0), (0, -1, 0), W, H, fovy_deg=40.0)
    if case == "depth_alpha":
        gD = rng.uniform(-1, 1, size=(H, W)).astype(np.float32)
        gA = rng.uniform(-1, 1, size=(H, W)).astype(np.float32)
    return cloud, cam, (0.2, 0.1, 0.3), gC, gD, gA


# ---- GPU ------------------------------------------------------------------------------------------------------------

def _subset(cloud, keep):
    return synth.Cloud(*(np.ascontiguousarray(a[keep]) for a in (cloud.means3D, cloud.scales, cloud.rotations,
                                                                  cloud.opacities, cloud.shs)), cloud.sh_degree)


def _gpu_radii(cloud, cam, colors_precomp=None, cov3D_precomp=None, scale_modifier=1.0):
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    ct = cloud_tensors(cloud, "cuda")
    rs = settings_from(cam, (0.0, 0.0, 0.0), cloud.sh_degree, "cuda", scale_modifier)
    kw = dict(means3D=ct["means3D"], means2D=torch.zeros_like(ct["means3D"]), opacities=ct["opacities"])
    if colors_precomp is not None:
        kw["colors_precomp"] = torch.from_numpy(colors_precomp).cuda()
    else:
        kw["shs"] = ct["shs"]
    if cov3D_precomp is not None:
        kw["cov3D_precomp"] = torch.from_numpy(cov3D_precomp).cuda()
    else:
        kw.update(scales=ct["scales"], rotations=ct["rotations"])
    with torch.no_grad():
        return GaussianRasterizer(rs)(**kw)[1].cpu().numpy()


def _matched(cloud, cam, colors_precomp=None, cov3D_precomp=None, scale_modifier=1.0):
    """Drops the rows whose radii differ between the GPU and the fp64 oracle (fp32 rounding and contraction at ceil(3
    sigma) or the near cut), then checks that both forwards agree on every radius. -> (cloud, cp, cov)."""
    def radii():
        f = O.forward_from(cloud, cam, f32=False, render=False, scale_modifier=scale_modifier,
                           **({} if colors_precomp is None else dict(colors_precomp=colors_precomp)),
                           **({} if cov3D_precomp is None else dict(cov3D_precomp=cov3D_precomp, scales=None,
                                                                    rotations=None)))
        r = f.radii.copy()
        f.close()
        return r, _gpu_radii(cloud, cam, colors_precomp, cov3D_precomp, scale_modifier)
    a, b = radii()
    keep = a == b
    if not keep.all():
        cloud = _subset(cloud, keep)
        colors_precomp = None if colors_precomp is None else np.ascontiguousarray(colors_precomp[keep])
        cov3D_precomp = None if cov3D_precomp is None else np.ascontiguousarray(cov3D_precomp[keep])
        a, b = radii()
    assert np.array_equal(a, b) and (a > 0).any()
    return cloud, colors_precomp, cov3D_precomp


def run_gpu(cloud, cam, bg, gC=None, gD=None, gA=None, colors_precomp=None, cov3D_precomp=None, scale_modifier=1.0,
            deterministic=False, static_capacity=None, sh_offset=False, settings=None):
    """One forward + backward with camera_grad=True -> dict(viewmatrix, projmatrix, campos, dmean3D) as float64."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    if settings is None:
        rs = settings_from(cam, bg, cloud.sh_degree, dev, scale_modifier)
        cam_t = {k: getattr(rs, k).clone().requires_grad_(True) for k in CAM}
        rs = rs._replace(**cam_t)
    else:
        rs, cam_t = settings, {}
    rast = GaussianRasterizer(rs, return_alpha=gA is not None, camera_grad=True, depth_grad=gD is not None,
                              deterministic=deterministic, static_capacity=static_capacity)
    kw = dict(means3D=ct["means3D"], means2D=torch.zeros_like(ct["means3D"], requires_grad=True),
              opacities=ct["opacities"])
    if colors_precomp is not None:
        kw["colors_precomp"] = torch.from_numpy(colors_precomp).to(dev).requires_grad_(True)
    elif sh_offset:   # the SH rows one float past a 16-byte boundary
        n = cloud.shs.size
        buf = torch.zeros(n + 4, dtype=torch.float32, device=dev)
        buf[1:n + 1] = torch.from_numpy(cloud.shs.reshape(-1)).to(dev)
        kw["shs"] = buf[1:n + 1].view(cloud.shs.shape)
        assert kw["shs"].data_ptr() % 16 == 4
    else:
        kw["shs"] = ct["shs"]
    if cov3D_precomp is not None:
        kw["cov3D_precomp"] = torch.from_numpy(cov3D_precomp).to(dev).requires_grad_(True)
    else:
        kw.update(scales=ct["scales"], rotations=ct["rotations"])
    out = rast(**kw)
    if static_capacity is not None:
        rast.check_capacity()
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    loss = 0.0
    if gC is not None:
        loss = loss + (out[0] * T(gC)).sum()
    if gD is not None:
        loss = loss + (out[2][0] * T(gD)).sum()
    if gA is not None:
        loss = loss + (out[3][0] * T(gA)).sum()
    loss.backward()
    got = {k: v.grad.detach().cpu().numpy().astype(np.float64) for k, v in cam_t.items()}
    dm = ct["means3D"].grad
    got["dmean3D"] = np.zeros(cloud.means3D.shape) if dm is None else dm.detach().cpu().numpy().astype(np.float64)
    return got


def check_camera(got, r, case, tau=TAU):
    """Element-wise |got - truth| <= tau B, relative L2 <= rho per array, exact zeros where nothing contributes."""
    stats = {}
    for name in CAM:
        g, want, B = got[name].reshape(r["B"][name].shape), r["truth"][name], r["B"][name]
        zero = B == 0
        assert not g[zero].any(), (case, name, g[zero])
        ratio = float((np.abs(g - want)[~zero] / B[~zero]).max()) if (~zero).any() else 0.0
        rel = rel_l2(g, want) if np.linalg.norm(want) > 0 else 0.0
        stats[name] = (ratio, rel)
        print(f"CAMSTAT {case} {name} max|got-truth|/B={ratio:.3e} relL2={rel:.3e}")
        assert ratio <= tau, (case, name, ratio)
        assert rel <= RHO[name], (case, name, rel)
    for name, idx in NEVER_READ.items():
        assert not got[name].reshape(4, 4)[idx].any(), (case, name)
    return stats


def check_identity(got, cam, case):
    s, mag = translation_identity(got["dmean3D"], got, cam.viewmatrix, cam.projmatrix)
    print(f"CAMSTAT {case} identity max|sum|/mag={float((np.abs(s) / mag).max()):.3e}")
    assert np.all(np.abs(s) <= TAU_ID * mag), (case, s, mag)


def _upstreams(cam, seed, depth=False, alpha=False):
    H, W = cam.image_height, cam.image_width
    rng = np.random.default_rng(seed)
    gC = rng.uniform(-0.5, 1.5, size=(3, H, W)).astype(np.float32)
    gD = rng.uniform(-0.3, 0.5, size=(H, W)).astype(np.float32) if depth else None
    gA = rng.uniform(-1.0, 1.0, size=(H, W)).astype(np.float32) if alpha else None
    return gC, gD, gA


def _compare(cloud, cam, case, bg=(0.2, 0.1, 0.3), depth=False, alpha=False, colors_precomp=None, cov3D_precomp=None,
             scale_modifier=1.0, seed=0, identity=True, tau=TAU, **gpu_kw):
    cloud, colors_precomp, cov3D_precomp = _matched(cloud, cam, colors_precomp, cov3D_precomp, scale_modifier)
    gC, gD, gA = _upstreams(cam, seed, depth, alpha)
    kw = dict(colors_precomp=colors_precomp, cov3D_precomp=cov3D_precomp, scale_modifier=scale_modifier)
    got = run_gpu(cloud, cam, bg, gC=gC, gD=gD, gA=gA, **kw, **gpu_kw)
    r = camera_truth(cloud, cam, bg, gC=gC, gD=gD, gA=gA, **kw)
    check_camera(got, r, case, tau)
    if identity:
        check_identity(got, cam, case)
    return got, r, cloud


def _base_cloud(P=20_000):
    cloud, _ = synth.make_config("c3", P=P)
    return cloud, synth.ring_cameras(8, 4.5, 15.0, 192, 144, 61.0)[5]


FORMS = {"deg0_M1": (0, 1), "deg1_M4": (1, 4), "deg2_M9": (2, 9), "deg3_M16": (3, 16), "deg1_M16": (1, 16),
         "deg0_M16": (0, 16), "colors_precomp": None, "sh_offset_M16": (3, 16)}


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [False, True], ids=["colour", "depth"])
@pytest.mark.parametrize("form", list(FORMS))
def test_kernel_forms(form, depth):
    """The four CAM instantiations ({bulk SH row, plain} x {with, without depth}) through every SH layout: degree 0-3,
    an active degree below the allocated one, colours precomputed (campos exactly 0), and an SH tensor one float past
    a 16-byte boundary."""
    cloud, cam = _base_cloud()
    cp = None
    if form == "colors_precomp":
        cp = np.random.default_rng(3).uniform(size=(cloud.means3D.shape[0], 3)).astype(np.float32)
    else:
        deg, M = FORMS[form]
        cloud.shs = np.ascontiguousarray(cloud.shs[:, :M, :])
        cloud.sh_degree = deg
    got, r, _ = _compare(cloud, cam, f"{form}/{'depth' if depth else 'colour'}", depth=depth, colors_precomp=cp,
                         sh_offset=form.startswith("sh_offset"), seed=1)
    if form == "colors_precomp" or form.startswith("deg0"):
        assert not got["campos"].any() and not r["truth"]["campos"].any()
    else:
        assert np.linalg.norm(r["truth"]["campos"]) > 0
    if depth:
        assert np.abs(r["g"]["ddepth"]).max() > 0


def _clamp_heavy(n=3000, seed=4):
    """Camera at the origin looking down +z; centres spread to |x/z|, |y/z| up to 2.2 tan(fov), large enough to reach
    into the frame from outside the clamp."""
    rng = np.random.default_rng(seed)
    cam = synth.look_at_camera((0, 0, 0), (0, 0, 1), (0, -1, 0), 160, 120, fovx_deg=50.0)
    z = rng.uniform(2.0, 6.0, n)
    r = rng.uniform(-2.2, 2.2, (n, 2)) * np.array([cam.tanfovx, cam.tanfovy])
    xyz = np.concatenate([r * z[:, None], z[:, None]], 1).astype(np.float32)
    scales = (z[:, None] * np.exp(rng.uniform(np.log(0.02), np.log(0.3), (n, 3)))).astype(np.float32)
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    sh = np.zeros((n, 16, 3), np.float32)
    sh[:, 0, :] = ((rng.uniform(size=(n, 3)) - 0.5) / 0.28209479177387814)
    sh[:, 1:, :] = rng.standard_normal((n, 15, 3)) * 0.1
    opac = rng.uniform(0.05, 0.9, (n, 1)).astype(np.float32)
    return synth.Cloud(xyz, scales, q.astype(np.float32), opac, sh.astype(np.float32), 3), cam


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["cov3D_precomp", "scale_modifier", "negative_dc", "return_alpha", "frustum_edge",
                                  "clamp_heavy"])
def test_other_inputs(case):
    kw = {}
    cloud, cam = _base_cloud()
    if case == "cov3D_precomp":
        f = O.forward_from(cloud, cam, render=False, f32=False)
        kw["cov3D_precomp"] = np.ascontiguousarray(f.cov3D.astype(np.float32))
        f.close()
    elif case == "scale_modifier":
        kw["scale_modifier"] = 0.7
    elif case == "negative_dc":
        cloud.shs[:, 0, :] -= np.float32(0.35 / 0.28209479177387814)
    elif case == "return_alpha":
        kw.update(depth=True, alpha=True)
    elif case == "frustum_edge":
        cloud, cam = synth.frustum_edge_cloud()
        kw.update(depth=True, tau=TAU_EDGE)
    else:
        cloud, cam = _clamp_heavy()
        kw["depth"] = True
    got, r, _ = _compare(cloud, cam, case, seed=2, **kw)
    if case == "negative_dc":
        assert r["rgb_clamped"].any(1).mean() >= 0.1, r["rgb_clamped"].any(1).mean()
    if case in ("clamp_heavy", "frustum_edge"):
        frac = r["clamped_xy"].mean()
        print(f"CAMSTAT {case} clamped fraction of the visible rows {frac:.3f} of {r['vis'].sum()}")
        assert frac >= (0.1 if case == "clamp_heavy" else 0.01), frac


BLOCKS = [(1, 96), (31, 31 * 128), (32, 32 * 128), (33, 32 * 128 + 96), (64, 64 * 128), (65, 64 * 128 + 100),
          (1025, 1025 * 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("nblocks,P", BLOCKS, ids=[f"{b}blocks_P{p}" for b, p in BLOCKS])
def test_block_counts(nblocks, P):
    """A 96-Gaussian visible scene padded IN FRONT with culled rows (behind the camera), so that the grid has nblocks
    blocks of 128 and the visible rows sit in the last block(s): from 33 blocks on, in blocks >= 32 only, so the
    strided part of the block-sum reduce carries the whole answer. Partial last blocks at 33 and 65."""
    assert (P + 127) // 128 == nblocks
    base, cam = _base_cloud(P=4000)
    f = O.forward_from(base, cam, render=False)
    vis = np.flatnonzero(f.radii > 0)[:96]
    f.close()
    small, _, _ = _matched(_subset(base, vis), cam)
    V = small.means3D.shape[0]
    pad = _subset(base, np.arange(P - V) % base.means3D.shape[0])
    fwd = cam.viewmatrix[:3, 2].astype(np.float64)          # camera z axis in world coordinates
    pad.means3D = (cam.campos[None, :] - (1.0 + (np.arange(P - V) % 7)[:, None]) * fwd[None, :]).astype(np.float32)
    cloud = synth.Cloud(*(np.concatenate([a, b]) for a, b in zip(
        (pad.means3D, pad.scales, pad.rotations, pad.opacities, pad.shs),
        (small.means3D, small.scales, small.rotations, small.opacities, small.shs))), base.sh_degree)
    assert cloud.means3D.shape[0] == P
    got, r, matched = _compare(cloud, cam, f"{nblocks}blocks", depth=True, seed=3)
    assert matched.means3D.shape[0] == cloud.means3D.shape[0]
    first_visible = int(np.flatnonzero(r["vis"])[0])
    assert nblocks <= 32 or first_visible // 128 >= 32, first_visible


@pytest.mark.gpu
def test_full_size_config3():
    """Config 3 camera 0: 1M Gaussians (7813 blocks), 1600x1200, against the fp64 oracle."""
    cloud, cams = synth.make_config("c3")
    assert (cloud.means3D.shape[0] + 127) // 128 == 7813
    _compare(cloud, cams[0], "c3_full", seed=4)


@pytest.mark.gpu
def test_deterministic_mode_and_static_capacity():
    """deterministic=True: the camera gradients repeat bit for bit and meet the bounds; the static-capacity form equals
    the default form bit for bit under deterministic mode."""
    cloud, cam = _base_cloud()
    cloud, _, _ = _matched(cloud, cam)
    gC, gD, _ = _upstreams(cam, 5, depth=True)
    bg = (0.2, 0.1, 0.3)
    a = run_gpu(cloud, cam, bg, gC=gC, gD=gD, deterministic=True)
    b = run_gpu(cloud, cam, bg, gC=gC, gD=gD, deterministic=True)
    s = run_gpu(cloud, cam, bg, gC=gC, gD=gD, deterministic=True, static_capacity=1 << 22)
    for k in CAM + ("dmean3D",):
        assert np.array_equal(a[k], b[k]), k
        assert np.array_equal(a[k], s[k]), k
    check_camera(a, camera_truth(cloud, cam, bg, gC=gC, gD=gD), "deterministic")
    check_identity(a, cam, "deterministic")


@pytest.mark.gpu
def test_empty_and_all_culled():
    cam = synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 64, 48, fovy_deg=50.0)
    gC = np.ones((3, 48, 64), np.float32)
    empty = synth.Cloud(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), np.zeros((0, 4), np.float32),
                        np.zeros((0, 1), np.float32), np.zeros((0, 16, 3), np.float32), 3)
    culled, _ = synth.make_config("c3", P=700)
    culled.means3D[:, 2] = -10.0
    for cloud in (empty, culled):
        for det in (False, True):
            got = run_gpu(cloud, cam, (0.3, 0.2, 0.1), gC=gC, gD=np.ones((48, 64), np.float32), deterministic=det)
            for k in CAM:
                assert got[k].shape == ((3,) if k == "campos" else (4, 4))
                assert not got[k].any(), (k, det)


@pytest.mark.gpu
def test_camera_grad_refuses_a_gradient_mask():
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    cloud, cam = _base_cloud(P=100)
    rs = settings_from(cam, (0, 0, 0), 3, "cuda")
    with pytest.raises(ValueError, match="camera_grad"):
        GaussianRasterizer(rs, camera_grad=True, grad_mask=torch.ones(100, dtype=torch.bool, device="cuda"))


def _rodrigues(w):
    th = torch.sqrt((w * w).sum())
    k = w / th
    K = torch.zeros(3, 3, dtype=w.dtype, device=w.device)
    K[0, 1], K[0, 2], K[1, 0], K[1, 2], K[2, 0], K[2, 1] = -k[2], k[1], k[2], -k[0], -k[1], k[0]
    return torch.eye(3, dtype=w.dtype, device=w.device) + torch.sin(th) * K + (1 - torch.cos(th)) * (K @ K)


def _pose_camera(pose, w2c0, projT):
    """GaussianEditor's camera from a 6-DoF pose (axis-angle, translation) applied on the left of a world-to-camera
    matrix: world_view_transform = W2C^T, full_proj_transform = world_view_transform @ projection^T, camera_center =
    world_view_transform.inverse()[3, :3]."""
    R = _rodrigues(pose[:3])
    top = torch.cat([R @ w2c0[:3, :3], (R @ w2c0[:3, 3] + pose[3:])[:, None]], 1)
    w2c = torch.cat([top, torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=pose.dtype, device=pose.device)], 0)
    view = w2c.transpose(0, 1)
    full = view.unsqueeze(0).bmm(projT.unsqueeze(0)).squeeze(0)
    return view, full, view.inverse()[3, :3]


@pytest.mark.gpu
def test_pose_chain():
    """pose.grad through the kernel's three gradients (the path a user takes: the camera arrays built from a pose with
    torch ops) equals the same chain in fp64 applied to the truth. Checks the layout and transposition of the returned
    .grad tensors."""
    cloud, cam = _base_cloud()
    pose_chain(cloud, cam, np.asarray(cam.viewmatrix, np.float64).T, np.array([0.02, -0.03, 0.015, 0.05, -0.02, 0.04]))


def pose_chain(cloud, cam, w2c0, p0, case="pose_chain"):
    """The camera of pose p0 (axis-angle, translation) applied to the world-to-camera matrix w2c0, with ``cam``'s frame
    and fields of view: pose.grad on the GPU against the fp64 chain of the truth."""
    projT = np.asarray(synth._projection(0.01, 100.0, cam.tanfovx, cam.tanfovy), np.float64).T
    pose = torch.tensor(p0, dtype=torch.float32, device="cuda", requires_grad=True)
    view, full, campos = _pose_camera(pose, torch.tensor(w2c0, dtype=torch.float32, device="cuda"),
                                      torch.tensor(projT, dtype=torch.float32, device="cuda"))
    pcam = synth.Camera(cam.image_height, cam.image_width, cam.tanfovx, cam.tanfovy,
                        view.detach().cpu().numpy().astype(np.float32), full.detach().cpu().numpy().astype(np.float32),
                        campos.detach().cpu().numpy().astype(np.float32))
    cloud, _, _ = _matched(cloud, pcam)
    bg = (0.2, 0.1, 0.3)
    gC, gD, _ = _upstreams(pcam, 6, depth=True)
    rs = settings_from(pcam, bg, cloud.sh_degree, "cuda")._replace(viewmatrix=view, projmatrix=full, campos=campos)
    run_gpu(cloud, pcam, bg, gC=gC, gD=gD, settings=rs)
    got = pose.grad.cpu().numpy().astype(np.float64)
    r = camera_truth(cloud, pcam, bg, gC=gC, gD=gD)

    def chain(p):
        v, f, c = _pose_camera(p, torch.tensor(w2c0), torch.tensor(projT))
        return torch.cat([v.reshape(-1), f.reshape(-1), c])
    J = torch.autograd.functional.jacobian(chain, torch.tensor(p0)).numpy()     # [35, 6]
    t = np.concatenate([r["truth"][k].reshape(-1) for k in CAM])
    B = np.concatenate([r["B"][k].reshape(-1) for k in CAM])
    want, Bp = J.T @ t, np.abs(J).T @ B
    ratio, rel = float((np.abs(got - want) / Bp).max()), rel_l2(got, want)
    print(f"CAMSTAT {case} max|got-truth|/B={ratio:.3e} relL2={rel:.3e}")
    assert ratio <= TAU and rel <= RHO_POSE, (case, got, want, ratio, rel)
