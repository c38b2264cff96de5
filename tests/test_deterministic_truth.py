"""Deterministic mode held to a truth, and the suite held to the shipped kernel options.

The deterministic backward stores one row per (instance, tile half) at the instance's emission slot with a flag, and
det_reduce_kernel (csrc/deterministic.cu) adds each Gaussian's run of flagged rows: runs of at most 64 rows by one
thread, longer runs by a whole warp. For the backward (two rows per instance) the switch lies between tiles_touched 32
and 33, for apply_weights (one row) between 64 and 65. A dropped or doubled row moves a gradient by a whole (pixel,
splat) contribution, so every check here is against a truth, not against the default path:
  * gradients of the colour, colour + depth and colour + alpha losses against the fp64 CPU oracle on the hard scenes, to
    the bound the default backward meets on each (5e-5; 1e-4 on the one-tile scenes, tests/test_list_edges.py), or,
    where the default backward on the same case is farther from fp64 than that, to its distance plus 1e-5;
  * on the needle scene, where fp32 and fp64 gradients part (the needle's conic is ill-conditioned), the per-Gaussian
    blend weight against the reference's recorded values: one dropped hit moves it by at least T/255;
  * a generated scene whose Gaussians touch 31..34, 63..66 and more than 1000 tiles, laid out so that 32-aligned index
    blocks (one warp of the reduction) hold several long runs and mix short and long ones;
  * apply_weights with masks in multiples of 2^-8 and every Gaussian's weight sum below 2^16, where every float sum is
    exact in any order: default, deterministic, sharded deterministic and the CPU oracle must agree bit for bit.

CPU: no test in tests/ changes a rasterizer option without restoring the value it found.
"""
import ast
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import _lib, synth
from util import cloud_tensors, rel_l2, settings_from

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPTIONS = ("render_fwd_variant", "render_bwd_variant", "preprocess_variant", "profile", "tile_key_bits",
           "binning_variant", "depth_sort_variant")


# ---------------------------------------------------------------------------------------------------------------- options
@pytest.fixture(scope="module", autouse=True)
def shipped_options():
    """The compiled defaults of every option, read in a fresh process, must be what this process holds: a test that
    leaves a variant switched would otherwise run every later test in the process on a kernel that does not ship."""
    code = ("import json; from gaussianeditor_b200 import _lib; L = _lib.load(); "
            f"print(json.dumps({{n: int(L.gsr_get_option(n.encode())) for n in {OPTIONS!r}}}))")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    shipped = json.loads(r.stdout.strip().splitlines()[-1])
    assert all(v >= 0 for v in shipped.values()), shipped
    lib = _lib.load()
    now = {n: int(lib.gsr_get_option(n.encode())) for n in OPTIONS}
    assert now == shipped, f"options left changed by an earlier test: {now} != shipped {shipped}"
    return shipped


_SETTERS = ("set_option", "gsr_set_option")


def _call_name(node):
    f = node.func
    return f.attr if isinstance(f, ast.Attribute) else f.id if isinstance(f, ast.Name) else None


def _calls(node, names):
    return [n for n in ast.walk(node) if isinstance(n, ast.Call) and _call_name(n) in names]


def option_leaks(source, filename="<test>"):
    """Line numbers of set_option / gsr_set_option calls in `source` that are neither inside the ``_options`` context
    manager nor covered by an explicit save and restore: in the same function, a name assigned from a gsr_get_option
    call, then a ``try`` whose ``finally`` sets an option from that name, with the call between the save and the end
    of that ``try``."""
    tree = ast.parse(source, filename)
    parent = {c: p for p in ast.walk(tree) for c in ast.iter_child_nodes(p)}
    leaks = []
    for call in _calls(tree, _SETTERS):
        chain, n = [], call
        while n in parent:
            n = parent[n]
            chain.append(n)
        if any(isinstance(a, ast.ClassDef) and a.name == "_options" for a in chain):
            continue
        func = next((a for a in chain if isinstance(a, (ast.FunctionDef, ast.AsyncFunctionDef))), None)
        ok = False
        if func is not None:
            saved = {}
            for a in ast.walk(func):
                if isinstance(a, (ast.Assign, ast.AnnAssign)) and a.value is not None and \
                        _calls(a.value, ("gsr_get_option",)):
                    for t in (a.targets if isinstance(a, ast.Assign) else [a.target]):
                        for nm in ast.walk(t):
                            if isinstance(nm, ast.Name):
                                saved.setdefault(nm.id, a.lineno)
            for t in ast.walk(func):
                if not isinstance(t, ast.Try) or not t.finalbody:
                    continue
                fin = ast.Module(body=t.finalbody, type_ignores=[])
                used = {nm.id for nm in ast.walk(fin) if isinstance(nm, ast.Name) and nm.id in saved}
                if not _calls(fin, _SETTERS) or not used:
                    continue
                if min(saved[u] for u in used) < call.lineno <= t.end_lineno:
                    ok = True
                    break
        if not ok:
            leaks.append(call.lineno)
    return leaks


def test_no_test_leaves_an_option_changed():
    found = {}
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "*.py"))):
        with open(path) as fh:
            lines = option_leaks(fh.read(), path)
        if lines:
            found[os.path.basename(path)] = lines
    assert not found, f"option changes without a restore (use test_parity_gpu._options): {found}"


def test_option_leak_check_sees_a_leak():
    leaky = ("def t():\n"
             "    _lib.set_option('render_bwd_variant', 4)\n"
             "    try:\n        run()\n"
             "    finally:\n        _lib.set_option('render_bwd_variant', 15)\n")
    assert option_leaks(leaky) == [2, 6]
    saved = ("def t():\n"
             "    old = lib.gsr_get_option(b'render_bwd_variant')\n"
             "    try:\n        lib.gsr_set_option(b'render_bwd_variant', 4)\n"
             "    finally:\n        lib.gsr_set_option(b'render_bwd_variant', old)\n"
             "    lib.gsr_set_option(b'render_bwd_variant', 4)\n")
    assert option_leaks(saved) == [7]


# ---------------------------------------------------------------------------------------------------------------- scenes
BOUNDARY_COUNTS = (31, 32, 33, 34, 63, 64, 65, 66)
HUGE = 1000


def _tiles_of(px, r, gx):
    """tiles_touched of a splat of integer radius r centred at pixel column px in a frame of one tile row (getRect)."""
    lo = np.clip(np.trunc((px - r) / 16.0), 0, gx)
    hi = np.clip(np.trunc((px + r + 15.0) / 16.0), 0, gx)
    return (hi - lo).astype(np.int64)


def boundary_cloud(seed=0):
    """Isotropic Gaussians in a 16400 x 16 frame (one row of 1025 tiles, so tiles_touched is the number of tile columns)
    -> (Cloud, Camera). Every count in BOUNDARY_COUNTS several times, a few Gaussians over more than HUGE tiles, and
    fillers of 1..8 tiles. Eight 32-aligned index blocks: all counts mixed; all 66 (32 long runs in one warp); fillers
    with two or three long runs; short/long neighbours 32|33 and 64|65 interleaved; the huge ones among fillers.

    Each splat's radius is set through its scale: 3 sqrt(lambda_max) = r - 0.5 (ceil gives r with half a unit to spare),
    and centres sit at half-pixels, so (p -+ r) / 16 stays half a pixel away from the tile edges whatever fp32 rounding
    the projection takes. Centres stay inside the frame: no Jacobian clamp."""
    rng = np.random.default_rng(seed)
    W, H = 16400, 16
    gx = (W + 15) // 16
    cam = synth._origin_camera(W, H)

    def place(target):
        while True:
            if target > HUGE:
                r = int(rng.integers(8300, 8600))
            elif target <= 8:
                r = int(rng.integers(8, 60))
            else:
                r = int(rng.integers(8 * target - 24, 8 * target + 8))
            px = float(rng.integers(0, W)) + 0.5
            if target <= 8 and 1 <= _tiles_of(np.array([px]), r, gx)[0] <= 8:
                return px, r
            if _tiles_of(np.array([px]), r, gx)[0] == target or (target > HUGE and _tiles_of(np.array([px]), r, gx)[0] > HUGE):
                return px, r

    mixed = lambda: list(rng.permutation(np.repeat(BOUNDARY_COUNTS, 4)))
    fill = lambda n: [1] * n
    blocks = [mixed(), [66] * 32, fill(30) + [33, 65], [32, 33] * 16, [64, 65] * 16, fill(29) + [34, 63, 66],
              fill(29) + [HUGE + 1] * 3, mixed()]
    blocks[2] = list(rng.permutation(blocks[2]))
    blocks[5] = list(rng.permutation(blocks[5]))
    blocks[6] = list(rng.permutation(blocks[6]))
    targets = [t for b in blocks for t in b]
    P = len(targets)
    px, r = np.array([place(t) for t in targets]).T
    py = np.full(P, 8.5)
    z = rng.permutation(np.linspace(3.0, 6.0, P))
    xyz = synth._at_pixels(cam, px, py, z)
    # lambda_max of s^2 J J^T + 0.3 with J J^T = (f/z)^2 [[1 + u^2, uv], [uv, 1 + v^2]]: eigenvalues (f/z)^2 and
    # (f/z)^2 (1 + u^2 + v^2); the reference takes mid + sqrt(max(0.1, spread^2))
    f = W / (2.0 * cam.tanfovx)
    w2 = (xyz[:, 0] ** 2 + xyz[:, 1] ** 2) / z ** 2
    lam = ((r - 0.5) / 3.0) ** 2
    a = (lam - 0.3) / (1.0 + w2)                               # spread above sqrt(0.1)
    small = a * w2 / 2.0 < np.sqrt(0.1)
    a = np.where(small, (lam - 0.3 - np.sqrt(0.1)) / (1.0 + w2 / 2.0), a)
    s = np.sqrt(a) * z / f
    opac = np.where(np.array(targets) > HUGE, rng.uniform(0.02, 0.05, P),
                    np.where(np.array(targets) <= 8, rng.uniform(0.1, 0.5, P), rng.uniform(0.05, 0.3, P)))
    cloud = synth.Cloud(xyz.astype(np.float32), np.repeat(s[:, None], 3, 1).astype(np.float32),
                        np.tile(np.array([[1.0, 0.0, 0.0, 0.0]], np.float32), (P, 1)), opac.astype(np.float32)[:, None],
                        synth._sh_dc(rng, P, 1), 1)
    return cloud, cam


def test_boundary_scene_hits_every_run_length():
    """On the CPU oracle's forward: every target count several times, the huge ones over HUGE tiles, and 32-aligned
    blocks holding two or more long runs of the backward (> 32 tiles) and of apply_weights (> 64 tiles) next to short
    ones."""
    from oracle import cpu_oracle
    cloud, cam = boundary_cloud()
    f = cpu_oracle.forward_from(cloud, cam, render=False)
    try:
        _check_run_lengths(f.tiles_touched.astype(np.int64))
    finally:
        f.close()


def _check_run_lengths(tt):
    for c in BOUNDARY_COUNTS:
        assert (tt == c).sum() >= 4, (c, (tt == c).sum())
    assert (tt > HUGE).sum() >= 3
    blocks = tt[: tt.size // 32 * 32].reshape(-1, 32)
    for cut in (32, 64):
        long_ = (blocks > cut).sum(1)
        assert ((long_ >= 2) & (long_ < 32)).sum() >= 3, (cut, long_)   # several long runs next to short ones
        assert (long_ == 32).any(), (cut, long_)                         # a warp of long runs only


_SCENES = {}


def _scene(name):
    """(cloud, cam, bg) by name, the last one kept."""
    if name not in _SCENES:
        bg = (0.1, 0.2, 0.3)
        if name == "needle":
            cloud, cam = synth.needle_cloud()
        elif name == "frustum_edge":
            cloud, cam = synth.frustum_edge_cloud()
        elif name == "opacity_edge":
            cloud, cam = synth.opacity_edge_cloud()
            bg = (0.0, 0.5, 1.0)
        elif name == "hotspot":
            cloud, cam = synth.hotspot_cloud()
        elif name == "tied_depth":
            cloud, cam = synth.tied_depth_cloud()
            bg = (0.3, 0.2, 0.1)
        elif name.startswith("one_tile/"):
            cloud, cam = synth.one_tile_cloud(int(name.split("/")[1]))
            bg = (0.0, 0.5, 1.0)
        elif name == "odd_333x201":
            cloud, _ = synth.make_config("c3", P=60_000)
            cam = synth.ring_cameras(8, 4.5, 15.0, 333, 201, 61.0)[5]
            bg = (0.2, 0.5, 0.7)
        elif name == "4112x4096":
            cloud, _ = synth.make_config("c3", P=20_000)
            cam = synth.ring_cameras(8, 4.5, 15.0, 4112, 4096, 61.0)[0]
        else:
            assert name == "boundary"
            cloud, cam = boundary_cloud()
        _SCENES.clear()
        _SCENES[name] = (cloud, cam, bg)
    return _SCENES[name]


# ---------------------------------------------------------------------------------------------------------------- GPU
def _run(cloud, cam, bg, gC, gD=None, gA=None, colors_precomp=None, grad_mask=None, deterministic=True):
    """Forward + backward through GaussianRasterizer; loss = sum gC*colour + sum gD*depth + sum gA*alpha. Returns
    (gradients under the CPU oracle's names, tiles_touched)."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians, forward_state_views
    dev = "cuda"
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    mask = None if grad_mask is None else torch.from_numpy(grad_mask).to(dev)
    rast = GaussianRasterizer(rs, return_alpha=gA is not None, depth_grad=gD is not None, deterministic=deterministic,
                              grad_mask=mask)
    kw = dict(means3D=ct["means3D"], means2D=m2, opacities=ct["opacities"], scales=ct["scales"],
              rotations=ct["rotations"])
    leaves = dict(dmean3D=ct["means3D"], dmean2D=m2, dopacity=ct["opacities"], dscale=ct["scales"],
                  drot=ct["rotations"])
    if colors_precomp is not None:
        kw["colors_precomp"] = leaves["dcolor"] = torch.from_numpy(colors_precomp).to(dev).requires_grad_(True)
    else:
        kw["shs"] = leaves["dsh"] = ct["shs"]
    out = rast(**kw)
    tt = forward_state_views(_RasterizeGaussians.last_state)["tiles_touched"].cpu().numpy().astype(np.int64)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    loss = (out[0] * T(gC)).sum()
    if gD is not None:
        loss = loss + (out[2][0] * T(gD)).sum()
    if gA is not None:
        loss = loss + (out[3][0] * T(gA)).sum()
    loss.backward()
    return {k: v.grad.detach().cpu().numpy() for k, v in leaves.items()}, tt


def _truth(cloud, cam, bg, form, gC, gD, f32=False):
    """fp64 gradients of the loss of `form`. colour: the oracle's backward. depth: test_depth_grad.depth_truth. alpha:
    sum gC*colour + sum gC[0]*alpha has the gradient of sum gC*colour with background (bg0 - 1, bg1, bg2), because
    colour_0 with that background is C_0 + alpha - 1 (test_parity_gpu: the alpha output test). ``f32=True``: the same
    on the fp32 oracle."""
    from oracle import cpu_oracle
    from test_depth_grad import depth_truth
    if form == "depth":
        g = depth_truth(cloud, cam, bg, gC=gC, gD=gD, f32=f32)
        g["fwd"].close()
        return g
    if form == "alpha":
        bg = (bg[0] - 1.0, bg[1], bg[2])
    f = cpu_oracle.forward_from(cloud, cam, bg, f32=f32)
    try:
        return f.backward(gC)
    finally:
        f.close()


def _upstreams(cam, seed):
    rng = np.random.default_rng(seed)
    H, W = cam.image_height, cam.image_width
    return rng.uniform(size=(3, H, W)).astype(np.float32), rng.uniform(-1, 1, size=(H, W)).astype(np.float32)


def _truth_errors(got, truth, skip=()):
    errs = {}
    for k, g in got.items():
        if k in skip:
            continue
        want = np.asarray(truth[k], np.float64)
        if np.linalg.norm(want) == 0:
            assert np.abs(g).max() == 0.0, k
            continue
        errs[k] = rel_l2(g.reshape(want.shape), want)
    return errs


def _check_truth(got, truth, tol, label, default=None, skip=()):
    """Relative L2 of every gradient from the fp64 truth <= tol. Where the default backward on the same case is itself
    farther than tol from the truth (`default`: its errors), the bound is its error plus 1e-5, the distance the
    deterministic backward may keep from the default (test_deterministic.py)."""
    errs = _truth_errors(got, truth, skip)
    d = default or {}
    bound = {k: d[k] + 1e-5 if d.get(k, 0.0) > tol else tol for k in errs}
    print(label, {k: f"{e:.2e}" + (f" (default {default[k]:.2e})" if default else "") for k, e in errs.items()},
          "bound", tol)
    bad = {k: (e, bound[k]) for k, e in errs.items() if not e <= bound[k]}
    assert not bad, (label, bad)


TRUTH_SCENES = ["frustum_edge", "opacity_edge", "hotspot", "tied_depth", "one_tile/33", "one_tile/4097",
                "odd_333x201", "4112x4096"]


def _truth_tol(scene):
    return 1e-4 if scene.startswith("one_tile") else 5e-5


# isotropic Gaussians: the rotation gradient is zero in exact arithmetic, both sides are rounding noise
_SKIP = {"boundary": ("drot",)}


def _against_truth(scene, form, seed=51):
    cloud, cam, bg = _scene(scene)
    gC, gD = _upstreams(cam, seed)
    kw = dict(gD=gD if form == "depth" else None, gA=gC[0] if form == "alpha" else None)
    got, tt = _run(cloud, cam, bg, gC, deterministic=True, **kw)
    default, _ = _run(cloud, cam, bg, gC, deterministic=False, **kw)
    truth = _truth(cloud, cam, bg, form, gC, gD)
    skip = _SKIP.get(scene, ())
    _check_truth(got, truth, _truth_tol(scene), (scene, form), _truth_errors(default, truth, skip), skip)
    return tt


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["colour", "depth", "alpha"])
@pytest.mark.parametrize("scene", TRUTH_SCENES)
def test_deterministic_backward_against_fp64(scene, form):
    """Every gradient of the deterministic backward against fp64, per tensor, to the scene's bound, or to the default
    backward's own distance plus 1e-5 where that is larger (the depth form on deep stacks). (The needle is checked per
    Gaussian below: its fp32 and fp64 gradients part by far more than any bound.)"""
    _against_truth(scene, form)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["colour", "depth"])
def test_boundary_scene_deterministic_against_fp64(form):
    """The run-length boundary scene: the forward's tiles_touched has every target count and the block layout; the
    deterministic backward against fp64."""
    tt = _against_truth("boundary", form)
    _check_run_lengths(tt)


def _needle_weights(deterministic=True, depth=False, masked=False, sharded=None):
    """Needle scene, precomputed colours, dL/dpixel = 1 on green: dcolor[:, 1] is each splat's total blend weight."""
    from test_parity_gpu import _needle_case
    cloud, cam, cp = _needle_case()
    H, W = cam.image_height, cam.image_width
    gC = np.zeros((3, H, W), np.float32)
    gC[1] = 1.0
    if sharded is not None:
        return _sharded_grads(cloud, cam, (0, 0, 0), gC, sharded, colors=cp)["colors"].cpu().numpy()
    P = cloud.means3D.shape[0]
    got, _ = _run(cloud, cam, (0, 0, 0), gC, gD=np.zeros((H, W), np.float32) if depth else None, colors_precomp=cp,
                  grad_mask=np.ones(P, np.uint8) if masked else None, deterministic=deterministic)
    return got["dcolor"]


def _check_needle_weights(got, label):
    """test_parity_gpu.test_needle_backward_blend_weights_every_variant's yardstick: the reference's dL_dcolors to 3x
    its run-to-run difference + 1e-5 relative + 1e-4."""
    from test_parity_gpu import _needle_case, _Ref, _ref_run
    cloud, cam, cp = _needle_case()
    dL = np.zeros((3, cam.image_height, cam.image_width), np.float32)
    dL[1] = 1.0

    def compute():
        a = _ref_run(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp)["grads"]["dL_dcolors"]
        b = _ref_run(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp)["grads"]["dL_dcolors"]
        return dict(dL_dcolors=a, noise=(a - b).abs())
    ref = _Ref("needle/bwd", compute, full=("dL_dcolors", "noise"))
    got = np.asarray(got, np.float64)
    want = np.asarray(ref.value("dL_dcolors"), np.float64).reshape(got.shape)
    noise = np.asarray(ref.value("noise"), np.float64).reshape(got.shape)
    tol = 3.0 * noise + 1e-5 * np.abs(want) + 1e-4
    assert np.all(got[:, [0, 2]] == 0.0) and (want[:, 1] > 0.0).mean() > 0.9
    over = np.abs(got - want) > tol
    print(label, "max |got - want| / tol", float((np.abs(got - want) / tol).max()))
    assert not over.any(), (label, np.argwhere(over)[:8].tolist(), np.abs(got - want)[over][:8])


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["plain", "depth", "grad_mask"])
def test_needle_blend_weights_deterministic(form):
    """Deterministic colour backward, its depth form with a zero depth upstream, and its masked form with every
    Gaussian under edit: each splat's blend weight equals the reference's, below half a dropped hit (T/255)."""
    _check_needle_weights(_needle_weights(depth=form == "depth", masked=form == "grad_mask"), form)


# ---- apply_weights with exact sums ---------------------------------------------------------------------------------
def _dyadic_mask(CH, H, W, seed):
    """Multiples of 2^-8 in [0, 63/256]: every partial sum of a Gaussian's weights is a multiple of 2^-8, and while
    hits * 63/256 < 2^16 it is exact in fp32, in any order of addition."""
    return (np.random.default_rng(seed).integers(0, 64, size=(CH, H, W)) / 256.0).astype(np.float32)


def _aw_inputs(cloud):
    t = cloud_tensors(cloud, "cuda")
    empty = torch.empty(0, device="cuda")
    return dict(means3D=t["means3D"], opacities=t["opacities"], shs=empty, colors=empty, scales=t["scales"],
                rotations=t["rotations"], cov=empty)


def _aw_gpu(cloud, cam, mask, deterministic):
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    d = _aw_inputs(cloud)
    P, CH = cloud.means3D.shape[0], mask.shape[0]
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
    w = torch.zeros(P, CH, device="cuda")
    c = torch.zeros(P, 1, dtype=torch.int32, device="cuda")
    GaussianRasterizer(rs, deterministic=deterministic).apply_weights(
        d["means3D"], None, d["opacities"], None, w, d["scales"], d["rotations"], None, c, torch.from_numpy(mask).cuda())
    return w.cpu(), c.cpu()


AW_SCENES = ["hotspot", "tied_depth", "needle", "boundary"]


@pytest.mark.gpu
@pytest.mark.parametrize("CH", [1, 2, 3])
@pytest.mark.parametrize("scene", AW_SCENES)
def test_apply_weights_exact_sums_agree_bit_for_bit(scene, CH):
    """Masks in multiples of 2^-8: default, deterministic and the sharded deterministic paths (dense and sparse, world 2
    and 3) give the same bits, and they equal the fp32 CPU oracle's on every Gaussian whose hit count the oracle
    shares; at most 1e-4 of the Gaussians may count differently (FMA contraction on the GPU). Not on the needle: there
    the hits along each needle's alpha = 1/255 contour depend on that rounding, and 43 % of its 1000 Gaussians count
    differently from the uncontracted oracle (measured on an H100); its forward is held bit-exact to the reference's
    CUDA build in test_parity_gpu.py."""
    from oracle import cpu_oracle
    from test_sharded_deterministic import _aw_dense, _aw_sparse
    cloud, cam, _ = _scene(scene)
    H, W = cam.image_height, cam.image_width
    P = cloud.means3D.shape[0]
    mask = _dyadic_mask(CH, H, W, seed=61 + CH)
    w0, c0 = _aw_gpu(cloud, cam, mask, False)
    assert int(c0.max()) // CH * float(mask.max()) < 1 << 16 and int((c0 > 0).sum()) > 0
    w1, c1 = _aw_gpu(cloud, cam, mask, True)
    assert torch.equal(c0, c1) and torch.equal(w0.view(torch.int32), w1.view(torch.int32))
    d = _aw_inputs(cloud)
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
    iw = torch.from_numpy(mask).cuda()
    for world in (2, 3):
        for name, (w, c) in (("dense", _aw_dense(world, rs, d, iw)), ("sparse", _aw_sparse(world, rs, d, iw, "tight"))):
            assert torch.equal(c.cpu(), c0), (name, world)
            assert torch.equal(w.cpu().view(torch.int32), w0.view(torch.int32)), (name, world)
    if scene == "boundary":   # runs on both sides of apply_weights' 64-row switch carried weight
        _, tt = _run(cloud, cam, (0, 0, 0), np.zeros((3, H, W), np.float32))
        for n in (64, 65):
            assert (w0.numpy()[tt == n] > 0).any(), n
    if scene == "needle":
        return
    f = cpu_oracle.forward_from(cloud, cam, colors_precomp=np.ones((P, 3), np.float32))
    try:
        wo = np.zeros((P, CH), np.float32)
        co = np.zeros((P, 1), np.int32)
        f.apply_weights(wo, co, mask)
    finally:
        f.close()
    same = (co == c0.numpy())[:, 0]
    assert (~same).mean() <= 1e-4, int((~same).sum())
    assert np.array_equal(w0.numpy()[same].view(np.int32), wo[same].view(np.int32))


# ---- sharded deterministic backward --------------------------------------------------------------------------------
def _sharded_grads(cloud, cam, bg, gC, spec, colors=None):
    """test_sharded_deterministic's virtual-rank drivers: spec = (path, world); the sparse path with tight segment
    capacity."""
    from test_sharded_deterministic import _dense_grads, _sparse_grads
    path, world = spec
    t = cloud_tensors(cloud, "cuda")
    empty = torch.empty(0, device="cuda")
    d = dict(means3D=t["means3D"], opacities=t["opacities"], shs=t["shs"] if colors is None else empty,
             colors=empty if colors is None else torch.from_numpy(colors).cuda(), scales=t["scales"],
             rotations=t["rotations"], cov=empty)
    rs = settings_from(cam, bg, cloud.sh_degree, "cuda")
    dL = torch.from_numpy(gC).cuda()
    if path == "dense":
        return _dense_grads(world, rs, d, dL)
    return _sparse_grads(world, rs, d, dL, "tight")


SHARD_SPECS = [("dense", 2), ("dense", 3), ("sparse", 2), ("sparse", 3)]
_SHARD_KEYS = dict(means3D="dmean3D", means2D="dmean2D", opacities="dopacity", scales="dscale", rotations="drot",
                   shs="dsh")


@pytest.mark.gpu
@pytest.mark.parametrize("path,world", SHARD_SPECS)
def test_sharded_deterministic_backward_against_truth(path, world):
    """The sharded deterministic backward: on the boundary scene every gradient against fp64 to 5e-5, on the needle
    every splat's blend weight against the reference's."""
    cloud, cam, bg = _scene("boundary")
    gC, gD = _upstreams(cam, 53)
    g = _sharded_grads(cloud, cam, bg, gC, (path, world))
    got = {_SHARD_KEYS[k]: v.cpu().numpy() for k, v in g.items()}
    _check_truth(got, _truth(cloud, cam, bg, "colour", gC, gD), _truth_tol("boundary"), ("boundary", path, world),
                 skip=_SKIP["boundary"])
    _check_needle_weights(_needle_weights(sharded=(path, world)), (path, world))
