"""Fused activations (``GaussianRasterizer.forward_raw``: gsr_backward_raw, gsr_backward_raw_depth and every other RAW
form, which share one chain-rule block) held to an fp64 truth of the functions they claim to apply.

The truth (``raw_truth``) takes the raw parameters in fp64, applies o = sigmoid(x), s = exp(ls), q = r / max(|r|, eps)
(eps = fp32(1e-12), F.normalize's) and sh = concat(dc, rest), rounds the activations to fp32, runs them through the
fp64 CPU oracle (``test_depth_grad.depth_truth`` when the loss has depth) and chains back in fp64:
sigmoid(x) sigmoid(-x), exp(ls), and (I - q q^T) / |r|, or I / eps where the norm was clamped.

CPU: the chain equals torch float64 autograd of the activations, and central fp64 finite differences of the oracle's
loss with respect to the raw parameters of isolated Gaussians.
GPU: each raw gradient's rel. L2 error against the truth (err_fused) is held to the error of the default path fed by
PyTorch's fp32 activations, with its activated gradients chained in fp64 (err_default): err_fused <= 2 err_default +
1e-6, and err_fused <= 5e-5 where the default path is within 2.5e-5 (``_compare``), on the rows whose radii agree
among the two calls and the oracle; deterministic mode unless a case says otherwise. Cases: every (degree, M)
GaussianEditor trains at, with P at and around multiples of the preprocess block; opaque logits in bands up to 18;
rotations negated, scaled by powers of two and with norms below eps; the depth gradient; the edge scenes.
"""
import os

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import synth
from oracle import cpu_oracle as O
from test_depth_grad import depth_truth
from util import rel_l2, settings_from

HERE = os.path.dirname(os.path.abspath(__file__))
EPS = float(np.float32(1e-12))      # F.normalize's eps as the kernels hold it: 1e-12f
KEYS = ("xyz", "opacity", "features_dc", "features_rest", "scaling", "rotation")


# ---- the fp64 truth ------------------------------------------------------------------------------------------------

def activations64(raw):
    """fp64 activations of the raw parameters (numpy fp32 dict keyed as KEYS)."""
    with np.errstate(over="ignore"):
        x = raw["opacity"].astype(np.float64)
        r = raw["rotation"].astype(np.float64)
        n = np.linalg.norm(r, axis=1)
        return dict(o=1.0 / (1.0 + np.exp(-x)), s=np.exp(raw["scaling"].astype(np.float64)),
                    q=r / np.maximum(n, EPS)[:, None], n=n,
                    sh=np.concatenate([raw["features_dc"], raw["features_rest"]], 1).astype(np.float64))


def cloud_of(raw, deg):
    """The activations rounded to fp32, as a synth.Cloud."""
    a = activations64(raw)
    f = lambda v: np.ascontiguousarray(v, np.float32)
    return synth.Cloud(f(raw["xyz"]), f(a["s"]), f(a["q"]), f(a["o"]), f(a["sh"]), deg)


def chain(raw, g):
    """Chain the activated gradients g (dmean3D, dopacity, dsh, dscale, drot) back to the raw parameters in fp64."""
    a = activations64(raw)
    x = raw["opacity"].astype(np.float64)
    with np.errstate(over="ignore"):
        dsig = (1.0 / (1.0 + np.exp(-x))) * (1.0 / (1.0 + np.exp(x)))    # sigmoid(x) sigmoid(-x): no 1 - o
    q, n = a["q"], a["n"]
    drot = np.asarray(g["drot"], np.float64).reshape(-1, 4)
    proj = (drot - q * (q * drot).sum(1, keepdims=True)) / np.maximum(n, EPS)[:, None]
    dsh = np.asarray(g["dsh"], np.float64)
    return dict(xyz=np.asarray(g["dmean3D"], np.float64).reshape(-1, 3),
                opacity=np.asarray(g["dopacity"], np.float64).reshape(-1, 1) * dsig,
                features_dc=dsh[:, :1], features_rest=dsh[:, 1:],
                scaling=np.asarray(g["dscale"], np.float64).reshape(-1, 3) * a["s"],
                rotation=np.where((n < EPS)[:, None], drot / EPS, proj))


def raw_truth(raw, deg, cam, bg, gC=None, gD=None):
    """fp64 gradients of  sum gC*colour + sum gD*depth  w.r.t. the raw parameters, and the oracle's radii."""
    g = depth_truth(cloud_of(raw, deg), cam, bg, gC=gC, gD=gD)
    radii = g["fwd"].radii.copy()
    g["fwd"].close()
    return chain(raw, g), radii


def to_raw(cloud, seed=0, max_shift=6):
    """A synth.Cloud in raw form: logits of the opacities, logs of the scales (an opacity of 1 or a scale of 0 gives an
    infinite logit or log), rotations times a random sign and power of two in 2^-max_shift..2^max_shift."""
    rng = np.random.default_rng(seed)
    P = cloud.means3D.shape[0]
    o = cloud.opacities.astype(np.float64)
    k = rng.integers(-max_shift, max_shift + 1, (P, 1)).astype(np.float64)
    with np.errstate(divide="ignore"):
        raw = dict(xyz=cloud.means3D, opacity=np.log(o) - np.log1p(-o), features_dc=cloud.shs[:, :1],
                   features_rest=cloud.shs[:, 1:], scaling=np.log(cloud.scales.astype(np.float64)),
                   rotation=cloud.rotations * np.where(rng.uniform(size=(P, 1)) < 0.5, -1.0, 1.0) * 2.0 ** k)
    return {kk: np.ascontiguousarray(v, np.float32) for kk, v in raw.items()}


# ---- CPU: the construction ------------------------------------------------------------------------------------------

def _chain_inputs(P=96, M=16, seed=0):
    rng = np.random.default_rng(seed)
    x = np.concatenate([np.linspace(-30.0, 30.0, 61), rng.normal(0.0, 4.0, P - 61)])
    r = rng.standard_normal((P, 4)) * np.exp(rng.uniform(-3.0, 3.0, (P, 1)))
    tiny = np.array([0.0, 1e-13, 5e-13, 9e-13, 3e-14, 2e-12, 1e-11])     # below, and a little above, eps
    r[: tiny.size] = r[: tiny.size] / np.linalg.norm(r[: tiny.size], axis=1, keepdims=True) * tiny[:, None]
    raw = dict(xyz=rng.standard_normal((P, 3)), opacity=x[:, None], features_dc=rng.standard_normal((P, 1, 3)),
               features_rest=rng.standard_normal((P, M - 1, 3)), scaling=rng.normal(-4.0, 1.0, (P, 3)), rotation=r)
    raw = {k: np.ascontiguousarray(v, np.float32) for k, v in raw.items()}
    g = dict(dmean3D=rng.standard_normal((P, 3)), dopacity=rng.standard_normal((P, 1)),
             dsh=rng.standard_normal((P, M, 3)), dscale=rng.standard_normal((P, 3)), drot=rng.standard_normal((P, 4)))
    return raw, g


def test_chain_matches_torch_autograd():
    """chain() against torch float64 autograd of sigmoid / exp / F.normalize / cat, logits in +-30, norms below eps
    and r = 0. Rows to 1e-12 relative. torch's sigmoid backward is o(1 - o), which in fp64 too keeps only an absolute
    accuracy of ~1e-16 as o -> 1: there the logit gradient is compared with that absolute bound, and every logit's
    against the closed form e^-|x| / (1 + e^-|x|)^2 to 1e-12 relative."""
    raw, g = _chain_inputs()
    ours = chain(raw, g)
    T = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    leaves = {k: T(raw[k]) for k in KEYS}
    o = torch.sigmoid(leaves["opacity"])
    s = torch.exp(leaves["scaling"])
    q = torch.nn.functional.normalize(leaves["rotation"], dim=1, eps=EPS)
    sh = torch.cat([leaves["features_dc"], leaves["features_rest"]], 1)
    G = lambda a: torch.tensor(np.asarray(a, np.float64))
    loss = ((leaves["xyz"] * G(g["dmean3D"])).sum() + (o * G(g["dopacity"])).sum() + (s * G(g["dscale"])).sum()
            + (q * G(g["drot"])).sum() + (sh * G(g["dsh"])).sum())
    loss.backward()
    for k in KEYS:
        want = leaves[k].grad.numpy()
        assert np.isfinite(ours[k]).all() and np.isfinite(want).all(), k
        if k == "opacity":
            assert np.all(np.abs(ours[k] - want) <= 1e-12 * np.abs(want) + 1e-15 * np.abs(g["dopacity"])), k
            continue
        a, b = ours[k].reshape(len(want), -1), want.reshape(len(want), -1)
        row = np.linalg.norm(a - b, axis=1) / np.maximum(np.linalg.norm(b, axis=1), 1e-300)
        assert row.max() <= 1e-12, (k, row.max())
    x = raw["opacity"].astype(np.float64)
    e = np.exp(-np.abs(x))
    closed = np.asarray(g["dopacity"]) * e / (1.0 + e) ** 2
    assert np.all(np.abs(ours["opacity"] - closed) <= 1e-12 * np.abs(closed)), "sigmoid derivative"
    # where the norm is clamped, F.normalize is r / eps: its derivative is I / eps, no projection
    n = np.linalg.norm(raw["rotation"].astype(np.float64), axis=1)
    assert (n < EPS).sum() == 5 and np.array_equal(ours["rotation"][n < EPS], np.asarray(g["drot"])[n < EPS] / EPS)
    # +-inf logits (an opacity of exactly 1 or 0): the derivative is 0, not NaN
    inf = dict(raw, opacity=np.array([[np.inf], [-np.inf]] + [[0.0]] * (len(x) - 2), np.float32))
    d = chain(inf, g)["opacity"]
    assert d[0, 0] == 0.0 and d[1, 0] == 0.0 and np.isfinite(d).all()


def _isolated_scene():
    """Six Gaussians on 64x48 pixels, far enough apart that their 3-sigma footprints do not meet; SH degree 3; logits
    -4, 9 and in -1.5..3, rotations of norm 0.3..3."""
    rng = np.random.default_rng(42)
    cam = synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 64, 48, fovy_deg=50.0)
    xy = np.array([[-0.9, -0.5], [0.0, -0.5], [0.9, -0.5], [-0.9, 0.5], [0.0, 0.5], [0.9, 0.5]])
    P = xy.shape[0]
    r = rng.standard_normal((P, 4))
    r *= rng.uniform(0.3, 3.0, (P, 1)) / np.linalg.norm(r, axis=1, keepdims=True)
    sh = rng.standard_normal((P, 16, 3)) * 0.3
    sh[:, 0, :] += 1.0
    logit = rng.uniform(-1.5, 3.0, (P, 1))
    logit[:2, 0] = (-4.0, 9.0)
    raw = dict(xyz=np.concatenate([xy, rng.uniform(-0.3, 0.3, (P, 1))], 1), opacity=logit, features_dc=sh[:, :1],
               features_rest=sh[:, 1:], scaling=np.log(rng.uniform(0.05, 0.1, (P, 3))), rotation=r)
    return {k: np.ascontiguousarray(v, np.float32) for k, v in raw.items()}, cam


def _raw_loss(raw64, cam, G, bg, g0):
    """The oracle's fp64 loss sum(colour * G) at fp64 raw parameters. The oracle takes the activations rounded to fp32;
    the rounding's first-order effect on the loss, sum g0 * (fp32(a) - a) with g0 the activated gradients at the
    unperturbed point, is taken off, so that what is left is the loss at the fp64 activations up to O(step * 6e-8)."""
    a = activations64(raw64)
    c = cloud_of(raw64, 3)
    f = O.forward_from(c, cam, bg, f32=False)
    loss = float((f.color * G).sum())
    nc, radii = f.n_contrib.copy(), f.radii.copy()
    f.close()
    loss -= float((g0["dopacity"] * (c.opacities - a["o"])).sum() + (g0["dscale"] * (c.scales - a["s"])).sum()
                  + (g0["drot"] * (c.rotations - a["q"])).sum() + (g0["dsh"] * (c.shs - a["sh"])).sum())
    return loss, nc, radii


def test_raw_truth_matches_fp64_finite_differences():
    """Directional central differences of the oracle's loss along random directions in each raw parameter of each
    isolated Gaussian, against raw_truth: the pattern and the 2e-4 bound of test_oracle_kat.py::
    test_gradients_match_fp64_finite_differences, with steps of 3e-4 and 1e-4 of the parameter's scale."""
    raw, cam = _isolated_scene()
    G = np.random.default_rng(7).uniform(size=(3, 48, 64)).astype(np.float32).astype(np.float64)
    bg = (0.3, 0.1, 0.6)
    truth, radii0 = raw_truth(raw, 3, cam, bg, gC=G.astype(np.float32))
    assert (radii0 > 0).all()
    f = O.forward_from(cloud_of(raw, 3), cam, bg, f32=False)
    g0 = f.backward(G.astype(np.float32))
    f.close()
    _, nc0, _ = _raw_loss(raw, cam, G, bg, g0)
    rng = np.random.default_rng(3)
    P = raw["xyz"].shape[0]
    for k in KEYS[1:]:
        ok = tried = 0
        for i in range(P):
            for trial in range(2):
                base = raw[k][i].astype(np.float64)
                d = rng.standard_normal(base.shape)
                d /= np.linalg.norm(d)
                scale = max(float(np.abs(base).max()), 1.0) if k != "rotation" else float(np.linalg.norm(base))
                for h in (3e-4, 1e-4):
                    plus, minus = dict(raw), dict(raw)
                    plus[k] = raw[k].astype(np.float64).copy(); plus[k][i] += h * scale * d
                    minus[k] = raw[k].astype(np.float64).copy(); minus[k][i] -= h * scale * d
                    l1, n1, r1 = _raw_loss(plus, cam, G, bg, g0)
                    l2, n2, r2 = _raw_loss(minus, cam, G, bg, g0)
                    if not (np.array_equal(r1, radii0) and np.array_equal(r2, radii0) and np.array_equal(n1, nc0)
                            and np.array_equal(n2, nc0)):
                        continue
                    tried += 1
                    ana = float((truth[k][i] * 2 * h * scale * d).sum())
                    if abs((l1 - l2) - ana) <= 2e-4 * abs(ana) + 1e-12:
                        ok += 1
        assert tried >= 12 and ok >= 0.7 * tried, (k, ok, tried)


# ---- GPU ------------------------------------------------------------------------------------------------------------

def _loss(out, gC, gD, dev):
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    loss = 0.0
    if gC is not None:
        loss = loss + (out[0] * T(gC)).sum()
    if gD is not None:
        loss = loss + (out[2][0] * T(gD)).sum()
    return loss


def run_fused(raw, deg, cam, bg, gC=None, gD=None, deterministic=None):
    """forward_raw + backward -> (colour, radii, depth) and the raw gradients, on the GPU."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    rast = GaussianRasterizer(settings_from(cam, bg, deg, dev), depth_grad=gD is not None, deterministic=deterministic)
    t = {k: torch.from_numpy(raw[k]).to(dev).requires_grad_(True) for k in KEYS}
    m2 = torch.zeros_like(t["xyz"], requires_grad=True)
    out = rast.forward_raw(means3D=t["xyz"], means2D=m2, opacity_logits=t["opacity"], features_dc=t["features_dc"],
                           features_rest=t["features_rest"], log_scales=t["scaling"], raw_rotations=t["rotation"])
    _loss(out, gC, gD, dev).backward()
    grads = {k: t[k].grad.cpu().numpy() for k in KEYS}
    grads["means2D"] = m2.grad.cpu().numpy()
    return [o.detach().cpu().numpy() for o in out], grads


def run_default(raw, deg, cam, bg, gC=None, gD=None, deterministic=None):
    """The default path on PyTorch's fp32 activations; its activated gradients chained in fp64 -> (radii, grads)."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    rast = GaussianRasterizer(settings_from(cam, bg, deg, dev), depth_grad=gD is not None, deterministic=deterministic)
    r = {k: torch.from_numpy(raw[k]).to(dev) for k in KEYS}
    leaf = lambda v: v.detach().contiguous().requires_grad_(True)
    xyz, op, sc = leaf(r["xyz"]), leaf(torch.sigmoid(r["opacity"])), leaf(torch.exp(r["scaling"]))
    rot = leaf(torch.nn.functional.normalize(r["rotation"]))
    sh = leaf(torch.cat((r["features_dc"], r["features_rest"]), dim=1))
    out = rast(means3D=xyz, means2D=torch.zeros_like(xyz), opacities=op, shs=sh, scales=sc, rotations=rot)
    _loss(out, gC, gD, dev).backward()
    g = dict(dmean3D=xyz.grad, dopacity=op.grad, dsh=sh.grad, dscale=sc.grad, drot=rot.grad)
    return out[1].cpu().numpy(), chain(raw, {k: v.cpu().numpy() for k, v in g.items()})


def _compare(raw, deg, cam, bg, gC=None, gD=None, bands=None, rows=None, deterministic=True):
    """The tolerance policy. ``bands``: {name: row mask}, each checked on its own (and "all" always); ``rows``: restrict
    every band to these rows. Returns the fused call's (outputs, grads).

    err_fused <= 2 err_default + 1e-6, and err_fused <= 5e-5 wherever the default path itself is within half of that
    (err_default <= 2.5e-5). Both calls share the blend backward, so in deterministic mode they sum every activated
    gradient in the same order and differ only where the activations or the chain rule do; in the atomic mode the
    order of the float atomics adds its own noise to both, independently. Where the fp32 forward misses the fp64 truth
    by more than the cap on both paths (a T < 1e-4 stop or an alpha threshold decided the other way in a few pixels of
    an opaque or ill-conditioned scene), the first bound alone holds the chain rule to the default path's accuracy."""
    out, fused = run_fused(raw, deg, cam, bg, gC, gD, deterministic)
    rad_d, dflt = run_default(raw, deg, cam, bg, gC, gD, deterministic)
    truth, rad_o = raw_truth(raw, deg, cam, bg, gC, gD)
    rad_f = out[1]
    P = rad_f.shape[0]
    agree = (rad_f == rad_d) & (rad_f == rad_o)
    assert (~agree).sum() <= 1e-4 * P, ("radii disagree", int((~agree).sum()), P)
    # culled rows, and coefficients above the active degree, are written as exact zeros
    for k in KEYS:
        assert np.isfinite(fused[k]).all(), k
        assert not fused[k][rad_f == 0].any(), k
    assert not fused["features_rest"][:, (deg + 1) ** 2 - 1:].any()
    bands = dict(bands or {})
    bands["all"] = np.ones(P, bool)
    fails, lines = [], []
    for name, m in bands.items():
        sel = m & agree & (rad_f > 0)
        if rows is not None:
            sel &= rows
        assert sel.sum() > 0, name
        for k in KEYS:
            t = truth[k][sel]
            if np.linalg.norm(t) == 0:
                assert not fused[k][sel].any(), (name, k)
                continue
            ef, ed = rel_l2(fused[k][sel], t), rel_l2(dflt[k][sel], t)
            capped = ed <= 2.5e-5
            lines.append(f"{name:>8} {k:>14}: err_fused {ef:.3e}  err_default {ed:.3e}  rows {int(sel.sum())}"
                         + ("" if capped else "  (default beyond the cap)"))
            if not (ef <= 2 * ed + 1e-6 and (ef <= 5e-5 or not capped)):
                fails.append(lines[-1])
    print("\n" + "\n".join(lines))
    assert not fails, "\n".join(fails)
    return out, fused


def _c3_raw(P, deg, M, seed=0):
    from test_parity_gpu import _raw_params
    cloud, _ = synth.make_config("c3", P=P)
    cloud.shs = np.ascontiguousarray(cloud.shs[:, :M, :])
    return {k: v.detach().numpy() for k, v in _raw_params(cloud, "cpu", seed).items()}


def _upstream(cam, seed, depth=False, colour=True):
    rng = np.random.default_rng(seed)
    H, W = cam.image_height, cam.image_width
    gC = rng.uniform(size=(3, H, W)).astype(np.float32) if colour else None
    gD = rng.uniform(-1, 1, size=(H, W)).astype(np.float32) if depth else None
    return gC, gD


CAM_SMALL = synth.ring_cameras(8, 4.5, 15.0, 160, 120, 61.0)[1]     # 120 rows: a partial last tile row


@pytest.mark.gpu
@pytest.mark.parametrize("P", [77, 2048, 2049, 2050, 2051, 2052, 2175])
@pytest.mark.parametrize("deg,M", [(0, 16), (1, 16), (2, 16), (3, 16), (0, 1), (1, 4), (2, 9)])
def test_degree_and_block_shape(deg, M, P):
    """P = 128k + r, r in {0, 1, 2, 3, 4, 127}, and P < 128: with M = 4 and 16 the last block of features_rest rows
    takes the bulk copy (r % 4 == 0) or the plain loads, in the forward and the backward."""
    raw = _c3_raw(P, deg, M)
    gC, _ = _upstream(CAM_SMALL, 5)
    _compare(raw, deg, CAM_SMALL, (0.3, 0.1, 0.2), gC=gC)


def _opaque_scene(deg=3, M=16, P=20_000):
    """A c3 cloud with a third of the logits uniform in [6, 18] (o up to 1 - 1.5e-8: a trained scene's opaque
    splats), at 192x144."""
    raw = _c3_raw(P, deg, M)
    rng = np.random.default_rng(17)
    pick = rng.permutation(P)[: P // 3]
    raw["opacity"][pick, 0] = rng.uniform(6.0, 18.0, pick.size).astype(np.float32)
    x = raw["opacity"][:, 0]
    bands = {"[6,9)": (x >= 6) & (x < 9), "[9,12)": (x >= 9) & (x < 12), "[12,18]": (x >= 12) & (x <= 18)}
    return raw, synth.ring_cameras(8, 4.5, 15.0, 192, 144, 61.0)[5], bands


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["deterministic", "atomic"])
def test_opaque_logits(mode):
    """sigmoid' as o(1 - o) in fp32 is off by 1e-5..1e-4 at logits 6..9, by 1e-2 at 12 and is exactly 0 from 16.7 on.
    Both backward modes: gsr_backward_raw_deterministic and gsr_backward_raw."""
    raw, cam, bands = _opaque_scene()
    gC, _ = _upstream(cam, 9)
    _compare(raw, 3, cam, (0.3, 0.1, 0.2), gC=gC, bands=bands, deterministic=mode == "deterministic")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["deterministic", "atomic"])
@pytest.mark.parametrize("loss", ["colour_depth", "depth"])
@pytest.mark.parametrize("deg", [3, 0])
def test_depth_grad_opaque(deg, loss, mode):
    """depth_grad on the opaque scene: gsr_backward_raw_deterministic with a depth upstream, and gsr_backward_raw_depth."""
    raw, cam, bands = _opaque_scene(deg, 16)
    gC, gD = _upstream(cam, 13, depth=True, colour=loss == "colour_depth")
    _compare(raw, deg, cam, (0.3, 0.1, 0.2), gC=gC, gD=gD, bands=bands, deterministic=mode == "deterministic")


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_rotation_sign_and_power_of_two_scale():
    """Deterministic mode. r -> -r keeps every output and gradient bit and negates d raw_rotations exactly.
    r -> 2^k r (|r|^2 stays a normal fp32 and |r| > eps) keeps every bit of the forward and of the other gradients and
    scales d raw_rotations by exactly 2^-k: the sum of squares scales by 4^k exactly through the fma chain, sqrtf by
    2^k, and __fdiv_rn(2^k r, 2^k n) = r / n."""
    raw = _c3_raw(5000, 3, 16)
    gC, _ = _upstream(CAM_SMALL, 19)
    bg = (0.3, 0.1, 0.2)
    out0, g0 = run_fused(raw, 3, CAM_SMALL, bg, gC, deterministic=True)
    assert (out0[1] > 0).sum() > 1000
    out1, g1 = run_fused(raw, 3, CAM_SMALL, bg, gC, deterministic=True)
    assert _same(out0, out1) and all(np.array_equal(g0[k], g1[k]) for k in g0)   # the premise: bit-reproducible
    out, g = run_fused(dict(raw, rotation=-raw["rotation"]), 3, CAM_SMALL, bg, gC, deterministic=True)
    assert _same(out, out0)
    assert np.array_equal(g["rotation"], -g0["rotation"])
    assert all(np.array_equal(g[k], g0[k]) for k in g0 if k != "rotation")
    n = np.linalg.norm(raw["rotation"].astype(np.float64), axis=1)
    for k in (-20, -3, 1, 7, 20):
        assert (n * 2.0 ** k).min() > 1e-12 and (n * 2.0 ** k).max() ** 2 < 1e38
        r = (raw["rotation"] * np.float32(2.0 ** k)).astype(np.float32)
        out, g = run_fused(dict(raw, rotation=r), 3, CAM_SMALL, bg, gC, deterministic=True)
        assert _same(out, out0), k
        assert np.array_equal(g["rotation"], (g0["rotation"] * np.float32(2.0 ** -k)).astype(np.float32)), k
        assert all(np.array_equal(g[kk], g0[kk]) for kk in g0 if kk != "rotation"), k


@pytest.mark.gpu
def test_rotation_norm_below_eps():
    """Visible Gaussians whose raw rotation has norm 0, 1e-13 or 5e-13: F.normalize divides by eps there, so the
    derivative is I / eps; the projection (I - q q^T) / |r| is off by |q|^2 = |r|^2 / eps^2 (1 % and 25 %)."""
    raw = _c3_raw(5000, 3, 16)
    gC, _ = _upstream(CAM_SMALL, 23)
    bg = (0.3, 0.1, 0.2)
    out, _ = run_fused(raw, 3, CAM_SMALL, bg, gC)
    rng = np.random.default_rng(29)
    vis = np.flatnonzero(out[1] >= 3)
    pick = rng.choice(vis, 90, replace=False)
    norms = np.repeat([0.0, 1e-13, 5e-13], 30)
    d = rng.standard_normal((90, 4))
    r = raw["rotation"].copy()
    r[pick] = (d / np.linalg.norm(d, axis=1, keepdims=True) * norms[:, None]).astype(np.float32)
    raw = dict(raw, rotation=r)
    rows = np.zeros(5000, bool)
    rows[pick] = True
    n = np.linalg.norm(r[pick].astype(np.float64), axis=1)
    assert (n < 1e-12).all() and (n[30:] > 0).all()
    out, _ = _compare(raw, 3, CAM_SMALL, bg, gC=gC, rows=rows)
    assert (out[1][pick] > 0).sum() >= 60


def _golden_hotspot():
    d = np.load(os.path.join(HERE, "golden", "hotspot_p1500_clones.npz"))
    cloud = synth.Cloud(d["means3D"], d["scales"], d["rotations"], d["opacities"], d["shs"], int(d["sh_degree"]))
    cam = synth.Camera(int(d["H"]), int(d["W"]), float(d["tanfovx"]), float(d["tanfovy"]), d["viewmatrix"],
                       d["projmatrix"], d["campos"])
    return cloud, cam


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["frustum_edge", "opacity_edge", "hotspot"])
def test_edge_scenes(scene):
    """Frustum edges (scales of exactly 0: log-scales of -inf), opacities at 1/255 and at and above 0.99 (an opacity
    of 1: logit +inf) and the hot-spot tile, in raw form, with a colour + depth loss. The needle scene is left out: its
    fp32 conic is too ill-conditioned for an fp64 yardstick (test_depth_grad.py::test_hard_scenes)."""
    if scene == "frustum_edge":
        cloud, cam = synth.frustum_edge_cloud()
    elif scene == "opacity_edge":
        cloud, cam = synth.opacity_edge_cloud()
    else:
        cloud, cam = _golden_hotspot()
    raw = to_raw(cloud, seed=31)
    gC, gD = _upstream(cam, 37, depth=True)
    _compare(raw, cloud.sh_degree, cam, (0.1, 0.2, 0.3), gC=gC, gD=gD)
