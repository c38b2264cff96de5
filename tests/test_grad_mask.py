"""Opt-in ``grad_mask``: gradients only for the Gaussians under edit (gsr_backward_masked / gsr_backward_raw_masked).

CPU: the new symbols are declared and exported, both entry points reject a NULL mask or a camera before touching a
device, the constructor checks dtype, shape, device and ``camera_grad``, the sharded rasterizer takes no mask, and the
deterministic MASK kernels contain no floating-point RED/ATOM.
GPU: in deterministic mode every masked row equals the unmasked deterministic backward's row bit for bit and every other
row is +0.0, for random, spatial, full, empty and culled-only masks, layered scenes with the edited layer in front of,
between and behind the others, the hot-spot golden cloud with half its clones masked, needle splats, an odd frame size
and P = 1, in every mode (SH, depth, alpha, colours, cov3D, fused activations with and without depth, static capacity
at R and overflowing). In the default atomic mode the masked rows are within rel. L2 1e-5 of the deterministic ones.
first[] of every tile equals a numpy restatement, and the edit-loop harness gives the same bits with the kernel mask as
with GaussianEditor's hooks, eagerly and in a CUDA graph.
"""
import ctypes as C
import functools
import inspect
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import _lib, synth
from util import cloud_tensors, rel_l2, settings_from

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "gsr_b200.h")
NEW_SYMBOLS = ("gsr_grad_mask_scratch_bytes", "gsr_backward_masked", "gsr_backward_raw_masked")
NONE = 0xFFFFFFFF   # GRAD_MASK_NONE: the tile has no edited instance


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_new_symbols_declared_and_exported():
    header = open(HEADER).read()
    lib = _lib.load()
    for name in NEW_SYMBOLS:
        assert re.search(r"GSR_API [^;]*\b%s\(" % name, header), name
        assert name in _lib.SYMBOLS and hasattr(lib, name), name
    assert lib.gsr_abi_version() == 2
    assert lib.gsr_grad_mask_scratch_bytes(1600, 1200) >= 100 * 75 * 4
    assert lib.gsr_grad_mask_scratch_bytes(0, 0) > 0


@pytest.mark.parametrize("entry", ["gsr_backward_masked", "gsr_backward_raw_masked"])
@pytest.mark.parametrize("bad", ["null_mask", "camera"])
def test_entry_points_reject_null_mask_and_camera(entry, bad):
    lib = _lib.load()
    fn = getattr(lib, entry)
    cam = _lib.CameraGrads()
    mask = (C.c_uint8 * 4)()
    args = [None] * len(fn.argtypes)
    sizes = [i for i, t in enumerate(fn.argtypes) if t is C.c_size_t or t is C.c_int32]
    for i in sizes:
        args[i] = 0
    i_cam = 16 if entry == "gsr_backward_masked" else 15
    i_mask = i_cam + 3
    args[i_cam] = C.byref(cam) if bad == "camera" else None
    args[i_mask] = C.cast(mask, C.c_void_p) if bad == "camera" else None
    rc = fn(*args)
    assert rc == -1
    msg = lib.gsr_last_error().decode()
    assert ("camera" in msg) if bad == "camera" else ("grad_mask" in msg), msg


def _rs():
    cam = synth.ring_cameras(1, 4.0, 10.0, 64, 48, 60.0)[0]
    return settings_from(cam, (0, 0, 0), 0, "cpu")


def test_constructor_validation():
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    rs = _rs()
    with pytest.raises(ValueError, match="bool or uint8"):
        GaussianRasterizer(rs, grad_mask=torch.ones(4, dtype=torch.float32))
    with pytest.raises(ValueError, match="1-D"):
        GaussianRasterizer(rs, grad_mask=torch.ones(2, 2, dtype=torch.bool))
    with pytest.raises(ValueError, match="device"):
        GaussianRasterizer(rs, grad_mask=torch.ones(4, dtype=torch.bool))   # a CPU tensor
    with pytest.raises(ValueError):
        GaussianRasterizer(rs, grad_mask=[1, 0, 1])
    assert GaussianRasterizer(rs).grad_mask is None


@pytest.mark.gpu
def test_constructor_validation_gpu():
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    cloud, cam = synth.make_config("c3", P=500)[0], synth.ring_cameras(1, 4.5, 15.0, 64, 48, 61.0)[0]
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
    m = torch.ones(500, dtype=torch.bool, device="cuda")
    with pytest.raises(ValueError, match="camera_grad"):
        GaussianRasterizer(rs, camera_grad=True, grad_mask=m)
    with pytest.raises(ValueError, match="contiguous"):
        GaussianRasterizer(rs, grad_mask=torch.ones(1000, dtype=torch.bool, device="cuda")[::2])
    r = GaussianRasterizer(rs, grad_mask=m)
    assert r.grad_mask.dtype == torch.uint8 and r.grad_mask.data_ptr() == m.data_ptr()   # a view, no copy
    ct = cloud_tensors(cloud, "cuda")
    r = GaussianRasterizer(rs, grad_mask=m[:499])
    with pytest.raises(ValueError, match="P = 500"):
        r(means3D=ct["means3D"], means2D=torch.zeros_like(ct["means3D"]), opacities=ct["opacities"], shs=ct["shs"],
          scales=ct["scales"], rotations=ct["rotations"])


def test_sharded_rasterizer_has_no_grad_mask():
    from gaussianeditor_b200.sharded import ShardedGaussianRasterizer
    assert "grad_mask" not in inspect.signature(ShardedGaussianRasterizer.__init__).parameters


def test_render_passes_grad_mask_only_when_given():
    from gaussianeditor_b200 import gaussian_renderer as GR
    src = inspect.getsource(GR.render)
    assert "grad_mask=None" in src and 'opt["grad_mask"] = grad_mask' in src


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="cuobjdump is not available")
def test_masked_det_kernels_have_no_float_atomics():
    lib_path = _lib.LIB_PATH
    if not os.path.exists(lib_path):
        pytest.skip("library not built")
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([exe, "-sass", lib_path], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            kernels[name].append(line.split("*/", 1)[1].split(";")[0].strip())
    # render_bwd_masked_kernel<MINB, DEPTH, DET>
    masked = {n: b for n, b in kernels.items() if re.search(r"render_bwd_masked_kernelILi\d+ELb[01]ELb[01]EEE", n)}
    det = {n: b for n, b in masked.items() if re.search(r"render_bwd_masked_kernelILi\d+ELb[01]ELb1EEE", n)}
    assert len(masked) == 4 and len(det) == 2, sorted(masked)
    assert any("grad_mask_first_kernel" in n for n in kernels)
    fatom = re.compile(r"^(?:@!?U?P\w+\s+)?(RED|ATOM)[GS]?\.\S*\.F(16|32|64)")
    for n, body in det.items():
        bad = [i for i in body if fatom.match(i)]
        assert not bad, (n, bad[:3])
    # the check would see them: the atomic masked kernels have them
    assert any(fatom.match(i) for n, b in masked.items() if n not in det for i in b)


# ---------------------------------------------------------------------------------------------------------------- GPU
MODES = ["sh", "depth", "alpha", "colors", "cov", "raw", "raw_depth", "static", "static_over"]


def _run(cloud, cam, mode, deterministic, mask=None, seed=0, bg=(0.1, 0.2, 0.3), capacity=None):
    """Forward + backward of one mode with an optional grad_mask (device bool [P]); (forward outputs, gradients) on the
    CPU, and the forward state."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians
    dev = "cuda"
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    H, W = cam.image_height, cam.image_width
    g = torch.Generator(device=dev).manual_seed(seed)
    up_c = torch.rand(3, H, W, generator=g, device=dev)
    up_d = torch.rand(1, H, W, generator=g, device=dev)
    up_a = torch.rand(1, H, W, generator=g, device=dev)
    means2D = torch.zeros_like(ct["means3D"], requires_grad=True)
    depth_grad = mode in ("depth", "raw_depth")
    opt = dict(return_alpha=mode == "alpha", depth_grad=depth_grad, deterministic=deterministic)
    if capacity is not None:
        opt["static_capacity"] = capacity
    if mask is not None:
        opt["grad_mask"] = mask
    rast = GaussianRasterizer(rs, **opt)
    leaves = {"means2D": means2D}
    if mode.startswith("raw"):
        shs = ct["shs"].detach()
        dc = shs[:, :1].clone().requires_grad_(True)
        rest = shs[:, 1:].clone().requires_grad_(True)
        logit = torch.logit(ct["opacities"].detach().clamp(1e-4, 1 - 1e-4)).requires_grad_(True)
        lsc = torch.log(ct["scales"].detach()).requires_grad_(True)
        rot = ct["rotations"].detach().clone().requires_grad_(True)
        out = rast.forward_raw(ct["means3D"], means2D, logit, dc, rest, lsc, rot)
        leaves.update(means3D=ct["means3D"], dc=dc, rest=rest, logit=logit, lsc=lsc, rot=rot)
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
            cp = torch.from_numpy(np.random.default_rng(seed).uniform(size=(cloud.means3D.shape[0], 3)).astype(np.float32))
            cp = cp.to(dev).requires_grad_(True)
            kw["colors_precomp"] = cp
            leaves["colors"] = cp
        else:
            kw["shs"] = ct["shs"]
            leaves["shs"] = ct["shs"]
        out = rast(**kw)
    state = _RasterizeGaussians.last_state
    loss = (out[0] * up_c).sum()
    if depth_grad:
        loss = loss + (out[2] * up_d).sum()
    if mode == "alpha":
        loss = loss + (out[3] * up_a).sum()
    loss.backward()
    fwd = {"color": out[0].detach().cpu(), "radii": out[1].cpu(), "depth": out[2].detach().cpu()}
    if mode == "alpha":
        fwd["alpha"] = out[3].detach().cpu()
    grads = {k: v.grad.detach().cpu().clone() for k, v in leaves.items() if v.grad is not None}
    return fwd, grads, state


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _capacity(cloud, cam, mode):
    """The static capacity of a static mode: R of a plain forward (exactly full), or R - 1 (overflowing); None for the
    other modes. Raises Skip when the frame has too few instances to overflow."""
    if not mode.startswith("static"):
        return None
    _, _, st = _run(cloud, cam, "sh", True)
    R = int(st.num_rendered)
    if mode == "static":
        return max(R, 1)
    if R < 2:
        pytest.skip("R < 2: no overflowing capacity")
    return R - 1


def _check_masked(cloud, cam, mode, mask):
    """Deterministic masked backward against the unmasked deterministic one: masked rows bit-identical, the others +0.0,
    forward outputs unchanged. Returns the masked run."""
    cap = _capacity(cloud, cam, mode)
    rmode = "sh" if mode.startswith("static") else mode
    ref_f, ref_g, _ = _run(cloud, cam, rmode, True, capacity=cap)
    got_f, got_g, state = _run(cloud, cam, rmode, True, mask=mask, capacity=cap)
    assert ref_f.keys() == got_f.keys()
    for k in ref_f:
        assert torch.equal(_bits(ref_f[k]), _bits(got_f[k])), k
    m = mask.cpu().bool()
    assert ref_g.keys() == got_g.keys()
    for k in ref_g:
        a, b = ref_g[k], got_g[k]
        assert a.shape == b.shape and a.shape[0] == m.numel(), k
        assert torch.equal(_bits(a[m]), _bits(b[m])), (k, "masked rows differ")
        assert bool((_bits(b[~m]) == 0).all()), (k, "unmasked rows are not +0.0")
    if mode == "static_over":   # an empty frame: zeros everywhere (the masked rows keep the unmasked signs of zero)
        for k, b in got_g.items():
            assert bool((b == 0).all()), k
    return got_f, got_g, state


@pytest.fixture(scope="module")
def small():
    cloud, _ = synth.make_config("c3", P=20_000)
    cam = synth.ring_cameras(8, 4.5, 15.0, 320, 240, 61.0)[0]
    return cloud, cam


def _mask(kind, cloud, cam, seed=0):
    P = cloud.means3D.shape[0]
    rng = np.random.default_rng(seed)
    if kind == "random30":
        m = rng.uniform(size=P) < 0.3
    elif kind == "spatial20":
        d = np.linalg.norm(cloud.means3D, axis=1)
        m = d <= np.quantile(d, 0.2)
    elif kind == "ones":
        m = np.ones(P, bool)
    elif kind == "zeros":
        m = np.zeros(P, bool)
    elif kind == "culled":
        _, _, st = _run(cloud, cam, "sh", True)
        m = (st.radii == 0).cpu().numpy()
        assert m.any() and not m.all()
    else:
        raise ValueError(kind)
    return torch.from_numpy(m).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["random30", "spatial20", "ones", "zeros", "culled"])
def test_masked_rows_bit_identical_small(small, kind, mode):
    cloud, cam = small
    mask = _mask(kind, cloud, cam)
    _, got_g, _ = _check_masked(cloud, cam, mode, mask)
    if kind == "zeros" or (kind == "culled" and mode != "cov"):   # cov3D_precomp culls a different set than SH + scales
        for k, b in got_g.items():
            assert bool((b == 0).all()), k


@pytest.mark.gpu
def test_uint8_mask_equals_bool_mask(small):
    cloud, cam = small
    m = _mask("random30", cloud, cam)
    _, a, _ = _run(cloud, cam, "sh", True, mask=m)
    _, b, _ = _run(cloud, cam, "sh", True, mask=m.to(torch.uint8) * 7)
    for k in a:
        assert torch.equal(_bits(a[k]), _bits(b[k])), k


def _layers(edited, per_layer=3000, seed=0):
    """Three overlapping layers at view depths 2, 4 and 6 over a 128x128 frame; the mask selects layer `edited`
    (0 = front, 1 = middle, 2 = back), so the early stop and the light path of the other layers are both exercised."""
    rng = np.random.default_rng(seed)
    cam = synth._origin_camera(128, 128)
    xyz, layer = [], []
    for i, z in enumerate((2.0, 4.0, 6.0)):
        xyz.append(synth._at_pixels(cam, rng.uniform(-4, 132, per_layer), rng.uniform(-4, 132, per_layer),
                                    np.full(per_layer, z) + rng.uniform(-0.2, 0.2, per_layer)))
        layer.append(np.full(per_layer, i))
    xyz = np.concatenate(xyz).astype(np.float32)
    layer = np.concatenate(layer)
    perm = rng.permutation(xyz.shape[0])   # layers interleaved in index
    xyz, layer = xyz[perm], layer[perm]
    P = xyz.shape[0]
    scales = (np.exp(rng.uniform(np.log(0.01), np.log(0.04), (P, 3))) * (xyz[:, 2:3] / 4.0)).astype(np.float32)
    q = rng.normal(size=(P, 4))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    opac = rng.uniform(0.2, 0.7, (P, 1)).astype(np.float32)
    shs = rng.uniform(-0.5, 0.5, (P, 4, 3)).astype(np.float32)
    cloud = synth.Cloud(xyz, scales, q, opac, shs, 1)
    return cloud, cam, torch.from_numpy(layer == edited).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("edited", [0, 1, 2])
def test_masked_layers(edited, mode):
    cloud, cam, mask = _layers(edited)
    _check_masked(cloud, cam, mode, mask)


def _golden_hotspot():
    d = np.load(os.path.join(HERE, "golden", "hotspot_p1500_clones.npz"))
    cloud = synth.Cloud(d["means3D"], d["scales"], d["rotations"], d["opacities"], d["shs"], int(d["sh_degree"]))
    cam = synth.Camera(int(d["H"]), int(d["W"]), float(d["tanfovx"]), float(d["tanfovy"]), d["viewmatrix"],
                       d["projmatrix"], d["campos"])
    P, base = cloud.means3D.shape[0], 1550   # 1500 hot-tile splats + 50 others, then the clones
    m = np.zeros(P, bool)
    m[base::2] = True                        # half of the clones: each shares its depth key with an unmasked row
    m[: base: 3] = True
    return cloud, cam, torch.from_numpy(m).cuda()


def _edge_scene(name):
    if name == "hotspot":
        return _golden_hotspot()
    if name == "needle":
        cloud, cam = synth.needle_cloud(P=600)
    elif name == "odd_frame":
        cloud, _ = synth.make_config("c3", P=8_000)
        cam = synth.ring_cameras(8, 4.5, 15.0, 333, 201, 61.0)[1]
    elif name == "p1":
        cam = synth._origin_camera(48, 40)
        xyz = synth._at_pixels(cam, np.array([20.0]), np.array([17.0]), np.array([3.0])).astype(np.float32)
        cloud = synth.Cloud(xyz, np.full((1, 3), 0.08, np.float32), np.array([[1, 0, 0, 0]], np.float32),
                            np.array([[0.8]], np.float32), np.full((1, 1, 3), 0.3, np.float32), 0)
        return cloud, cam, torch.ones(1, dtype=torch.bool, device="cuda")
    else:
        raise ValueError(name)
    m = np.random.default_rng(3).uniform(size=cloud.means3D.shape[0]) < 0.5
    return cloud, cam, torch.from_numpy(m).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("scene", ["hotspot", "needle", "odd_frame", "p1"])
def test_masked_edge_scenes(scene, mode):
    cloud, cam, mask = _edge_scene(scene)
    _check_masked(cloud, cam, mode, mask)
    if scene == "p1":   # and the single Gaussian unmasked: all zeros
        _, g, _ = _run(cloud, cam, "sh" if mode.startswith("static") else mode, True, mask=~mask)
        for k, b in g.items():
            assert bool((_bits(b) == 0).all()), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sh", "depth", "alpha", "colors", "raw", "raw_depth"])
@pytest.mark.parametrize("kind", ["random30", "spatial20", "ones"])
def test_atomic_mode_close_to_deterministic(small, kind, mode):
    cloud, cam = small
    mask = _mask(kind, cloud, cam)
    _, det, _ = _run(cloud, cam, mode, True, mask=mask)
    _, ato, _ = _run(cloud, cam, mode, False, mask=mask)
    m = mask.cpu()
    for k in det:
        assert bool((_bits(ato[k][~m]) == 0).all()), k
        if det[k][m].abs().max() > 0:
            assert rel_l2(ato[k][m].numpy(), det[k][m].numpy()) <= 1e-5, k


@pytest.mark.gpu
def test_torch_deterministic_flag_selects_det_masked(small):
    cloud, cam = small
    mask = _mask("random30", cloud, cam)
    _, det, _ = _run(cloud, cam, "sh", True, mask=mask)
    torch.use_deterministic_algorithms(True)
    try:
        _, flag, _ = _run(cloud, cam, "sh", None, mask=mask)
    finally:
        torch.use_deterministic_algorithms(False)
    for k in det:
        assert torch.equal(_bits(det[k]), _bits(flag[k])), k


def _first_restated(state, mask):
    """first[] of every tile from the binning and image views: the 1-based position of the first instance whose
    Gaussian is masked among positions [0, min(tile_last, list length)), tile_last = max n_contrib of the tile."""
    from gaussianeditor_b200.rasterizer import forward_state_views
    v = forward_state_views(state)
    W, H = state.W, state.H
    gx, gy = (W + 15) // 16, (H + 15) // 16
    nc = np.zeros((gy * 16, gx * 16), np.int64)
    nc[:H, :W] = v["n_contrib"].cpu().numpy()
    tile_last = nc.reshape(gy, 16, gx, 16).max(axis=(1, 3)).reshape(-1)
    ranges = v["ranges"].cpu().numpy().astype(np.int64)
    pl = v["point_list"].cpu().numpy().astype(np.int64)
    m = mask.cpu().numpy().astype(bool)
    out = np.full(gx * gy, NONE, np.uint32)
    for t in range(gx * gy):
        a, b = ranges[t]
        n = min(tile_last[t], max(b - a, 0))
        hit = np.nonzero(m[pl[a:a + n]])[0]
        if hit.size:
            out[t] = hit[0] + 1
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["small_random30", "small_spatial20", "layers_back", "hotspot", "odd_frame"])
def test_grad_mask_first_matches_restatement(small, scene):
    if scene.startswith("small"):
        cloud, cam = small
        mask = _mask(scene.split("_")[1], cloud, cam)
    elif scene == "layers_back":
        cloud, cam, mask = _layers(2)
    else:
        cloud, cam, mask = _edge_scene(scene)
    _, _, state = _run(cloud, cam, "sh", True, mask=mask)
    ntile = ((state.W + 15) // 16) * ((state.H + 15) // 16)
    got = state.mask_first.view(torch.int32)[:ntile].cpu().numpy().view(np.uint32)
    want = _first_restated(state, mask)
    assert np.array_equal(got, want), np.nonzero(got != want)[0][:10]
    assert (want != NONE).any() and (want != 1).any()


def _loop(mode, cuda_graph):
    from gaussianeditor_b200.edit_loop import run_edit_loop
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    return run_edit_loop(functools.partial(GaussianRasterizer, deterministic=True), steps=200, P=200_000, densification_interval=100, deterministic=True,
                         grad_mask=mode, cuda_graph=cuda_graph)


@pytest.mark.gpu
@pytest.mark.parametrize("cuda_graph", [False, True])
def test_edit_loop_kernel_mask_equals_hooks(cuda_graph):
    a = _loop("hooks", cuda_graph)
    b = _loop("kernel", cuda_graph)
    assert a["counts"] == b["counts"] and a["counts"][0] != a["counts"][-1]   # one densification
    assert np.array_equal(np.array(a["losses"], np.float32).view(np.int32), np.array(b["losses"], np.float32).view(np.int32))
    for n in a["params"]:
        assert torch.equal(_bits(a["params"][n]), _bits(b["params"][n])), n
    pa = [p for g in a["optimizer"].param_groups for p in g["params"]]
    pb = [p for g in b["optimizer"].param_groups for p in g["params"]]
    for x, y in zip(pa, pb):
        sa, sb = a["optimizer"].state[x], b["optimizer"].state[y]
        assert sa.keys() == sb.keys()
        for k in sa:
            assert torch.equal(_bits(torch.as_tensor(sa[k]).float()), _bits(torch.as_tensor(sb[k]).float())), k
