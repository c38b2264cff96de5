"""Deterministic mode: bit-reproducible gradients and apply_weights without float atomics.

CPU: the DET kernels contain no floating-point RED/ATOM; the emission-slot formula the deterministic backward stores its
rows at maps the instances one-to-one onto [0, R) in the binning's emission order, checked on the CPU oracle's forward
state; the sharded rasterizer refuses torch's deterministic flag.
GPU: two calls give the same bits (every backward combination, several scenes, frame sizes, binning / depth-sort
variants, the speculative forward, apply_weights, two processes, the edit loop); values stay within the default
path's. Anything that sets torch's flag runs in a subprocess.
"""
import json
import os
import re
import shutil
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import _lib, synth
from util import cloud_tensors, rel_l2, settings_from

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gaussianeditor_b200", "csrc", "libgsr_b200.so")


def _run_py(code, env_extra=None, timeout=1800):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    env.update(env_extra or {})
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=timeout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="cuobjdump is not available")
def test_det_kernels_have_no_float_atomics():
    if not os.path.exists(LIB):
        pytest.skip("library not built")
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            kernels[name].append(line.split("*/", 1)[1].split(";")[0].strip())
    # render_bwd_flat_kernel<NSB, MINB, SKIP, MASKSKIP, BATCHED, DEPTH, DET = true>
    det_bwd = re.compile(r"render_bwd_flat_kernelI(?:Li\d+E){2}(?:Lb[01]E){4}Lb1EEE")
    is_det = lambda n: bool(det_bwd.search(n)) or any(k in n for k in ("AwDetArgs", "det_reduce_kernel", "det_excl_kernel"))
    det = {n: b for n, b in kernels.items() if is_det(n)}
    # colour and depth backward, apply_weights for 1..3 channels, 5 reductions, the prefix scatter
    assert len([n for n in det if det_bwd.search(n)]) == 2 and len([n for n in det if "AwDetArgs" in n]) == 3
    assert len(det) == 11, sorted(det)
    fatom = re.compile(r"^(?:@!?U?P\w+\s+)?(RED|ATOM)[GS]?\.\S*\.F(16|32|64)")
    for n, body in det.items():
        bad = [i for i in body if fatom.match(i)]
        assert not bad, (n, bad[:3])
    # the check would see them: the default backward has them
    assert any(fatom.match(i) for n, b in kernels.items() if "render_bwd_flat_kernel" in n for i in b)


def _slots_from_oracle(f, gx, gy):
    """(instance tile, Gaussian) of the oracle's sorted list and the emission slot of each by the formula of
    common.cuh: emission_slot, with excl from the (depth bits, index) order the forward's depth sort produces."""
    P = f.P
    depth_bits = f.depths.astype(np.float32).view(np.uint32).astype(np.uint64)
    touched = f.tiles_touched.astype(np.int64)
    key = np.where(touched > 0, depth_bits, np.uint64(0xFFFFFFFF))
    order = np.lexsort((np.arange(P), key))
    excl = np.zeros(P, np.int64)
    excl[order] = np.cumsum(touched[order]) - touched[order]
    tile_of = np.zeros(f.num_rendered, np.int64)
    for t, (a, b) in enumerate(f.ranges):
        tile_of[a:b] = t
    g = f.point_list.astype(np.int64)
    px = f.means2D[g, 0].astype(np.float32); py = f.means2D[g, 1].astype(np.float32)
    rad = f.radii[g].astype(np.float32)
    T = np.float32(16)
    trunc = lambda v: np.trunc(v).astype(np.int64)
    rminx = np.clip(trunc((px - rad) / T), 0, gx); rminy = np.clip(trunc((py - rad) / T), 0, gy)
    rmaxx = np.clip(trunc((px + rad + np.float32(15)) / T), 0, gx)
    tx, ty = tile_of % gx, tile_of // gx
    slot = excl[g] + (ty - rminy) * (rmaxx - rminx) + (tx - rminx)
    return slot, g, tile_of, order, excl


@pytest.mark.parametrize("scene", ["c3_small", "frustum_edge", "needle", "hotspot", "tied_depth"])
def test_emission_slots_are_a_bijection_in_emission_order(scene):
    """hotspot: one tile list of ~70 000 instances; tied_depth: ~27 000 visible Gaussians sharing one depth key (excl
    follows the index order inside the tie) and exact copies far apart in index."""
    from oracle import cpu_oracle
    if scene == "c3_small":
        cloud, cams = synth.make_config("c3", P=3000)
        cam = cams[0]
    elif scene == "frustum_edge":
        cloud, cam = synth.frustum_edge_cloud()
    elif scene == "hotspot":
        cloud, cam = synth.hotspot_cloud()
    elif scene == "tied_depth":
        cloud, cam = synth.tied_depth_cloud()
    else:
        cloud, cam = synth.needle_cloud(P=300)
    f = cpu_oracle.forward_from(cloud, cam)
    try:
        R = f.num_rendered
        assert R > 0
        gx, gy = (f.W + 15) // 16, (f.H + 15) // 16
        slot, g, tile, order, excl = _slots_from_oracle(f, gx, gy)
        # one-to-one onto [0, R)
        assert np.array_equal(np.sort(slot), np.arange(R))
        # each Gaussian owns [excl, excl + tiles_touched) and within it the instances come in duplicateWithKeys'
        # order: the tile rectangle row by row (its position relative to the reference's point_offsets)
        off_excl = f.point_offsets.astype(np.int64) - f.tiles_touched.astype(np.int64)
        inv = np.empty(R, np.int64)
        inv[slot] = np.arange(R)
        g_by_slot, tile_by_slot = g[inv], tile[inv]
        # Gaussians appear in depth order, each one's tiles row-major (what the reference emits per Gaussian)
        rank = np.empty(f.P, np.int64)
        rank[order] = np.arange(f.P)
        assert np.all(np.diff(rank[g_by_slot]) >= 0)
        same = g_by_slot[1:] == g_by_slot[:-1]
        assert np.all(np.diff(tile_by_slot)[same] > 0)
        # relative position of every instance inside its Gaussian's run equals the reference's emission position
        ref_pos = np.zeros(R, np.int64)
        by_g = np.lexsort((tile, g))      # per Gaussian, its instances by tile
        ref_pos[by_g] = np.arange(R) - np.searchsorted(g[by_g], g[by_g], side="left")
        assert np.array_equal(slot - excl[g], ref_pos)
        assert np.all(off_excl[g] + ref_pos < f.point_offsets[g])
        if scene == "frustum_edge":   # clamped rectangles are part of this scene
            assert np.any(f.means2D[f.radii > 0, 0] - f.radii[f.radii > 0] < 0)
    finally:
        f.close()


def test_sharded_rasterizer_refuses_torch_deterministic_flag():
    out = _run_py("""
        import warnings, torch
        from gaussianeditor_b200 import sharded
        torch.use_deterministic_algorithms(True)
        try:
            sharded.ShardedGaussianRasterizer.forward(None, None, None, None)
        except RuntimeError as e:
            assert "deterministic" in str(e), e
            print("raised")
        torch.use_deterministic_algorithms(True, warn_only=True)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            sharded._check_deterministic_flag()
        assert any("deterministic" in str(x.message) for x in w)
        print("warned")
    """)
    assert "raised" in out and "warned" in out


# ---------------------------------------------------------------------------------------------------------------- GPU
MODES = ["sh", "colors", "cov", "alpha", "camera", "depth", "camera_depth", "raw", "raw_depth"]


def _grads(cloud, cam, mode, deterministic, seed=0, bg=(0.1, 0.2, 0.3)):
    """Forward + backward of one mode; returns (forward outputs, gradients) as CPU tensors."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    dev = "cuda"
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    H, W = cam.image_height, cam.image_width
    g = torch.Generator(device=dev).manual_seed(seed)
    up_c = torch.rand(3, H, W, generator=g, device=dev)
    up_d = torch.rand(1, H, W, generator=g, device=dev)
    up_a = torch.rand(1, H, W, generator=g, device=dev)
    means2D = torch.zeros_like(ct["means3D"], requires_grad=True)
    depth_grad = mode in ("depth", "camera_depth", "raw_depth")
    camera = mode in ("camera", "camera_depth")
    if camera:
        rs = rs._replace(viewmatrix=rs.viewmatrix.clone().requires_grad_(True),
                         projmatrix=rs.projmatrix.clone().requires_grad_(True),
                         campos=rs.campos.clone().requires_grad_(True))
    rast = GaussianRasterizer(rs, return_alpha=mode == "alpha", camera_grad=camera, depth_grad=depth_grad,
                              deterministic=deterministic)
    leaves = {"means2D": means2D}
    if mode.startswith("raw"):
        P = ct["means3D"].shape[0]
        shs = ct["shs"].detach()
        dc = shs[:, :1].clone().requires_grad_(True)
        rest = shs[:, 1:].clone().requires_grad_(True)
        logit = torch.logit(ct["opacities"].detach().clamp(1e-4, 1 - 1e-4)).requires_grad_(True)
        lsc = torch.log(ct["scales"].detach()).requires_grad_(True)
        rot = ct["rotations"].detach().clone().requires_grad_(True)
        m3 = ct["means3D"]
        out = rast.forward_raw(m3, means2D, logit, dc, rest, lsc, rot)
        leaves.update(means3D=m3, dc=dc, rest=rest, logit=logit, lsc=lsc, rot=rot)
    else:
        kw = dict(means3D=ct["means3D"], means2D=means2D, opacities=ct["opacities"])
        leaves.update(means3D=ct["means3D"], opacities=ct["opacities"])
        if mode == "cov":
            s = ct["scales"].detach()
            cov = torch.zeros(s.shape[0], 6, device=dev)
            cov[:, 0], cov[:, 3], cov[:, 5] = s[:, 0] ** 2, s[:, 1] ** 2, s[:, 2] ** 2
            cov.requires_grad_(True)
            kw["cov3D_precomp"] = cov
            leaves["cov"] = cov
        else:
            kw.update(scales=ct["scales"], rotations=ct["rotations"])
            leaves.update(scales=ct["scales"], rotations=ct["rotations"])
        if mode == "colors":
            cp = torch.from_numpy(np.random.default_rng(seed).uniform(size=(cloud.means3D.shape[0], 3)).astype(np.float32)).to(dev)
            cp.requires_grad_(True)
            kw["colors_precomp"] = cp
            leaves["colors"] = cp
        else:
            kw["shs"] = ct["shs"]
            leaves["shs"] = ct["shs"]
        out = rast(**kw)
    loss = (out[0] * up_c).sum()
    if depth_grad:
        loss = loss + (out[2] * up_d).sum()
    if mode == "alpha":
        loss = loss + (out[3] * up_a).sum()
    loss.backward()
    if camera:
        leaves.update(view=rs.viewmatrix, proj=rs.projmatrix, campos=rs.campos)
    fwd = {"color": out[0].detach().cpu(), "radii": out[1].cpu(), "depth": out[2].detach().cpu()}
    if mode == "alpha":
        fwd["alpha"] = out[3].detach().cpu()
    grads = {k: v.grad.detach().cpu().clone() for k, v in leaves.items() if v.grad is not None}
    return fwd, grads


def _bits_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].numpy().tobytes() == b[k].numpy().tobytes(), k


def _small_scene():
    cloud, cams = synth.make_config("c3", P=20_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 320, 240, 61.0)[0]
    return cloud, cam


@pytest.fixture(scope="module")
def small():
    return _small_scene()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_repeatable_and_close_to_default_small(small, mode):
    cloud, cam = small
    f1, g1 = _grads(cloud, cam, mode, True)
    f2, g2 = _grads(cloud, cam, mode, True)   # the second call takes the speculative forward (capacity hint)
    _bits_equal(g1, g2)
    _bits_equal(f1, f2)
    f0, g0 = _grads(cloud, cam, mode, False)
    _bits_equal(f0, f1)                       # forward outputs do not depend on the mode
    for k in g0:
        assert rel_l2(g1[k].numpy(), g0[k].numpy()) <= 1e-5, (k, rel_l2(g1[k].numpy(), g0[k].numpy()))


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["needle", "frustum_edge", "opacity_edge"])
def test_repeatable_edge_scenes(scene):
    if scene == "needle":
        cloud, cam = synth.needle_cloud()
    elif scene == "frustum_edge":
        cloud, cam = synth.frustum_edge_cloud()
    else:
        cloud, cam = synth.opacity_edge_cloud()
    for mode in ("sh", "depth"):
        _, g1 = _grads(cloud, cam, mode, True)
        _, g2 = _grads(cloud, cam, mode, True)
        _bits_equal(g1, g2)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(1, 1), (17, 9), (4112, 4096)])
@pytest.mark.parametrize("binning,depth_sort", [(1, 0), (0, 1)])
def test_repeatable_frame_sizes_and_variants(size, binning, depth_sort):
    W, H = size
    cloud, _ = synth.make_config("c3", P=20_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, W, H, 61.0)[0]
    old = {n: int(_lib.load().gsr_get_option(n.encode())) for n in ("binning_variant", "depth_sort_variant")}
    try:
        _lib.set_option("binning_variant", binning)
        _lib.set_option("depth_sort_variant", depth_sort)
        det = {}
        for mode in ("sh", "depth"):
            _, det[mode] = _grads(cloud, cam, mode, True)
            _, g2 = _grads(cloud, cam, mode, True)
            _bits_equal(det[mode], g2)
        _, g0 = _grads(cloud, cam, "sh", False)
        for k in g0:
            assert rel_l2(det["sh"][k].numpy(), g0[k].numpy()) <= 1e-5 or not g0[k].abs().sum() > 0, k
    finally:
        for n, v in old.items():
            _lib.set_option(n, v)


@pytest.mark.gpu
def test_speculative_forward_is_taken_and_repeatable(small):
    from gaussianeditor_b200 import rasterizer as RZ
    cloud, cam = small
    n0 = RZ.SPEC_STATS["launched"]
    _, g1 = _grads(cloud, cam, "sh", True)
    _, g2 = _grads(cloud, cam, "sh", True)
    assert RZ.SPEC_STATS["launched"] > n0
    assert RZ._RasterizeGaussians.last_state.cap > RZ._RasterizeGaussians.last_state.num_rendered
    _bits_equal(g1, g2)


@pytest.mark.gpu
def test_close_to_fp64_oracle(small):
    from oracle import cpu_oracle
    cloud, cam = small
    bg = (0.1, 0.2, 0.3)
    dL = np.random.default_rng(0).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    ct = cloud_tensors(cloud, "cuda", requires_grad=True)
    rs = settings_from(cam, bg, cloud.sh_degree, "cuda")
    m2 = torch.zeros_like(ct["means3D"], requires_grad=True)
    color, _, _ = GaussianRasterizer(rs, deterministic=True)(means2D=m2, **ct)
    (color * torch.from_numpy(dL).cuda()).sum().backward()
    f = cpu_oracle.forward_from(cloud, cam, bg, f32=False)
    try:
        g = f.backward(dL)
        ours = dict(dmean3D=ct["means3D"].grad, dmean2D=m2.grad, dopacity=ct["opacities"].grad, dscale=ct["scales"].grad,
                    drot=ct["rotations"].grad, dsh=ct["shs"].grad)
        for k, v in ours.items():
            assert rel_l2(v.cpu().numpy(), g[k]) <= 2e-4, (k, rel_l2(v.cpu().numpy(), g[k]))
    finally:
        f.close()


def _apply_weights(cloud, cams, deterministic, n_views=None, rounds=1):
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    ct = cloud_tensors(cloud, "cuda")
    P = cloud.means3D.shape[0]
    weights = torch.zeros(P, 1, device="cuda")
    cnt = torch.zeros(P, 1, dtype=torch.int32, device="cuda")
    for _ in range(rounds):
        for i, cam in enumerate(cams[:n_views]):
            rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
            H, W = cam.image_height, cam.image_width
            yy, xx = torch.meshgrid(torch.arange(H, device="cuda"), torch.arange(W, device="cuda"), indexing="ij")
            mask = (((xx - W / 2) ** 2 + (yy - H / 2) ** 2) < (0.3 * min(W, H)) ** 2).float()[None]
            GaussianRasterizer(rs, deterministic=deterministic).apply_weights(
                ct["means3D"], None, ct["opacities"], None, weights, ct["scales"], ct["rotations"], None, cnt, mask)
    return weights.cpu(), cnt.cpu()


@pytest.mark.gpu
def test_apply_weights_repeatable_and_close():
    cloud, cams = synth.make_config("c5")
    w1, c1 = _apply_weights(cloud, cams, True, n_views=4)
    w2, c2 = _apply_weights(cloud, cams, True, n_views=4)
    assert torch.equal(w1.view(torch.int32), w2.view(torch.int32)) and torch.equal(c1, c2)
    w0, c0 = _apply_weights(cloud, cams, False, n_views=4)
    assert torch.equal(c0, c1)
    assert rel_l2(w1.numpy(), w0.numpy()) <= 1e-6
    assert (w1 > 0).sum() > 1000


@pytest.mark.gpu
def test_apply_weights_48_views_twice_same_mask():
    cloud, cams = synth.make_config("c5")
    masks = []
    for _ in range(2):
        w, c = _apply_weights(cloud, cams, True, rounds=1)
        masks.append((w / c.clamp_min(1)) > 0.5)
    assert torch.equal(masks[0], masks[1]) and masks[0].sum() > 0


DIGEST = """
    import hashlib, json, numpy as np, torch
    from gaussianeditor_b200 import synth
    from test_deterministic import _grads
    cloud, cams = synth.make_config("c3")
    out = {}
    for mode in ("sh", "depth"):
        _, g = _grads(cloud, cams[0], mode, True)
        out.update({f"{mode}/{k}": hashlib.sha256(v.numpy().tobytes()).hexdigest() for k, v in g.items()})
    print("DIGESTS", json.dumps(out, sort_keys=True))
"""


@pytest.mark.gpu
def test_config3_digests_equal_across_processes():
    runs = [_run_py(DIGEST) for _ in range(2)]
    d = [json.loads(r.split("DIGESTS", 1)[1]) for r in runs]
    assert d[0] == d[1] and len(d[0]) >= 12


FLAG = """
    import functools, hashlib, json, os, sys, numpy as np, torch
    import torch.utils.deterministic
    from types import SimpleNamespace
    from gaussianeditor_b200 import gaussian_renderer as GR, synth, edit_loop, optim_surgery
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    mode = sys.argv[-1] if len(sys.argv) > 1 else ""
    if os.environ.get("DET_FLAG") == "1":
        torch.use_deterministic_algorithms(True)
        torch.utils.deterministic.fill_uninitialized_memory = True
    explicit = {} if os.environ.get("DET_FLAG") == "1" else {"deterministic": True}
    cloud, cams = synth.make_config("c5", P=50_000)
    scene = edit_loop.EditScene(cloud, "cuda")
    view = edit_loop.make_view(cams[0], "cuda")
    pipe = SimpleNamespace(convert_SHs_python=False, compute_cov3D_python=False, debug=False)
    bg = torch.zeros(3, device="cuda")
    pkg = GR.render(view, scene, pipe, bg, **explicit)
    g = torch.Generator(device="cuda").manual_seed(0)
    (pkg["render"] * torch.rand(pkg["render"].shape, generator=g, device="cuda")).sum().backward()
    out = {"render": pkg["render"].detach(), "vsp": pkg["viewspace_points"].grad,
           **{n: getattr(scene, n).grad for n in ("_xyz", "_opacity", "_features_dc", "_features_rest", "_scaling",
                                                   "_rotation")}}
    w = torch.zeros(scene._xyz.shape[0], 1, device="cuda"); c = torch.zeros(scene._xyz.shape[0], 1, dtype=torch.int32, device="cuda")
    H, W = cams[0].image_height, cams[0].image_width
    iw = torch.ones(1, H, W, device="cuda")
    rast = GaussianRasterizer(GR._settings_for(view, bg, 1.0, scene.active_sh_degree), **explicit)
    rast.apply_weights(scene.get_xyz, None, scene.get_opacity, None, w, scene.get_scaling, scene.get_rotation, None, c, iw)
    out["weights"] = w; out["cnt"] = c
    print("DIGESTS", json.dumps({k: hashlib.sha256(v.detach().cpu().numpy().tobytes()).hexdigest()
                                 for k, v in out.items()}, sort_keys=True))
"""


@pytest.mark.gpu
def test_torch_flag_selects_deterministic_path_without_reading_uninitialised_memory():
    env = {"CUBLAS_WORKSPACE_CONFIG": ":4096:8"}
    flagged = json.loads(_run_py(FLAG, dict(env, DET_FLAG="1")).split("DIGESTS", 1)[1])
    explicit = json.loads(_run_py(FLAG, dict(env, DET_FLAG="0")).split("DIGESTS", 1)[1])
    assert flagged == explicit


EDIT = """
    import functools, json, torch
    from gaussianeditor_b200.edit_loop import run_edit_loop
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    r = run_edit_loop(functools.partial(GaussianRasterizer, deterministic=True), steps=200)
    import hashlib
    print("RESULT", json.dumps({"counts": r["counts"], "losses": [float(x).hex() for x in r["losses"]],
                                "radii": hashlib.sha256(r["max_radii2D"].numpy().tobytes()).hexdigest()}))
"""


@pytest.mark.gpu
def test_edit_loop_twice_identical():
    runs = [json.loads(_run_py(EDIT).split("RESULT", 1)[1]) for _ in range(2)]
    assert runs[0] == runs[1] and len(runs[0]["counts"]) == 200
