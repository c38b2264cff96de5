"""Opt-in ``mask_render``: the image of the masked Gaussians drawn in white, written by the colour pass itself.

GaussianEditor renders every camera twice per step; the second forward draws the edit mask in white
(``render(..., override_color=mask.float()[:, None].repeat(1, 3))["render"]``) and only thresholds it. With
``GaussianRasterizer(mask_render=mask)`` the first forward returns that image as a trailing output, bit for bit, from the
same blend walk (render_fwd_mask_kernel, gsr_forward_*_mask). These tests hold it to the second forward's bits on every
forward form, and hold every other output and gradient to the same call without the option.
"""
import ctypes as C
import glob
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
TWINS = ("gsr_forward_render_mask", "gsr_forward_render_speculative_mask", "gsr_forward_static_mask",
         "gsr_forward_static_raw_mask")
CUOBJDUMP = shutil.which("cuobjdump") or ("/usr/local/cuda/bin/cuobjdump"
                                          if os.path.exists("/usr/local/cuda/bin/cuobjdump") else None)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_new_symbols_declared_exported_and_bound():
    header = open(HEADER).read()
    lib = _lib.load()
    for name in TWINS:
        assert re.search(r"GSR_API [^;]*\b%s\(" % name, header), name
        assert name in _lib.SYMBOLS and hasattr(lib, name), name
        # the twin's arguments are its base entry point's, plus (mask, out_mask_render) before the stream
        base = getattr(lib, name[:-len("_mask")]).argtypes
        assert list(getattr(lib, name).argtypes) == list(base[:-1]) + [C.c_void_p] * 3, name
    assert lib.gsr_abi_version() == 2


@pytest.mark.parametrize("entry", TWINS)
@pytest.mark.parametrize("bad", ["mask", "out"])
def test_entry_points_reject_null_mask_or_output_before_any_device_work(entry, bad):
    lib = _lib.load()
    fn = getattr(lib, entry)
    args = [None] * len(fn.argtypes)
    for i, t in enumerate(fn.argtypes):
        if t is C.c_size_t or t is C.c_int32:
            args[i] = 0
    host = (C.c_uint8 * 16)()   # never dereferenced: the check comes first
    args[-3] = None if bad == "mask" else C.cast(host, C.c_void_p)
    args[-2] = C.cast(host, C.c_void_p) if bad == "mask" else None
    assert fn(*args) == -1
    msg = lib.gsr_last_error().decode()
    assert "mask_render" in msg and (("mask is null" in msg) if bad == "mask" else ("out_mask_render" in msg)), msg


def _rs():
    cam = synth.ring_cameras(1, 4.0, 10.0, 64, 48, 60.0)[0]
    return settings_from(cam, (0, 0, 0), 0, "cpu")


def test_constructor_validation():
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    rs = _rs()
    with pytest.raises(ValueError, match="mask_render must be a bool or uint8"):
        GaussianRasterizer(rs, mask_render=torch.ones(4, dtype=torch.float32))
    with pytest.raises(ValueError, match="mask_render must be 1-D"):
        GaussianRasterizer(rs, mask_render=torch.ones(2, 2, dtype=torch.bool))
    with pytest.raises(ValueError, match="mask_render must be on the rasterizer's CUDA device"):
        GaussianRasterizer(rs, mask_render=torch.ones(4, dtype=torch.bool))
    with pytest.raises(ValueError, match="mask_render"):
        GaussianRasterizer(rs, mask_render=torch.ones(8, dtype=torch.bool)[::2])   # non-contiguous (and on the CPU)
    with pytest.raises(ValueError, match="mask_render must be a torch.Tensor"):
        GaussianRasterizer(rs, mask_render=[1, 0, 1])
    # the grad_mask messages are unchanged
    with pytest.raises(ValueError, match="^grad_mask must be a bool or uint8 tensor"):
        GaussianRasterizer(rs, grad_mask=torch.ones(4, dtype=torch.float32))
    r = GaussianRasterizer(rs)
    assert r.mask_render is None and r.grad_mask is None


def test_render_passes_mask_render_only_when_given(monkeypatch):
    from gaussianeditor_b200 import gaussian_renderer as GR
    seen = []

    class Recorder:   # a stand-in with the reference's constructor: fails on any keyword it does not know
        def __init__(self, raster_settings, **kw):
            seen.append(kw)
            raise RuntimeError("stop")

    monkeypatch.setattr(GR, "GaussianRasterizer", Recorder)
    pc = type("PC", (), {"get_xyz": torch.zeros(3, 3), "active_sh_degree": 0})()
    view = type("V", (), dict(image_height=48, image_width=64, FoVx=1.0, FoVy=0.8,
                              world_view_transform=torch.eye(4), full_proj_transform=torch.eye(4),
                              camera_center=torch.zeros(3)))()
    for kw in ({}, {"mask_render": torch.ones(3, dtype=torch.bool)}):
        with pytest.raises(RuntimeError, match="stop"):
            GR.render(view, pc, None, torch.zeros(3), **kw)
    assert seen[0] == {} and list(seen[1]) == ["mask_render"]
    assert "mask_render=None" in inspect.getsource(GR.render)


# the render_fwd kernels of the parent build, by their mangled names past the file's anonymous namespace
OLD_KERNELS = ("render_fwd_cta_kernelENS0_10RenderArgsE",
               "render_fwd_warp_kernelILi8ELb0ELb0EEEvNS0_10RenderArgsEi",
               "render_fwd_warp_kernelILi4ELb1ELb0EEEvNS0_10RenderArgsEi",
               "render_fwd_warp_kernelILi4ELb0ELb0EEEvNS0_10RenderArgsEi",
               "render_fwd_warp_kernelILi2ELb0ELb0EEEvNS0_10RenderArgsEi",
               "render_fwd_warp_kernelILi2ELb0ELb1EEEvNS0_10RenderArgsEi",
               "render_fwd_packed_kernelENS0_10RenderArgsEi")
MASK_KERNEL = "render_fwd_mask_kernelENS0_10RenderArgsEiPKhPf"


@pytest.mark.skipif(CUOBJDUMP is None, reason="cuobjdump is not available")
def test_render_fwd_kernels_keep_their_names_and_the_mask_kernel_is_built():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    sass = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    names = set(re.findall(r"Function : (\S+)", sass))
    fwd = {re.sub(r"^.*render_fwd_cu_[0-9a-f]+_?\d+", "", n) for n in names if "render_fwd_cu" in n}
    for k in OLD_KERNELS + (MASK_KERNEL,):
        assert k in fwd, (k, sorted(fwd))
    assert "sm_90a" in sass


# ---------------------------------------------------------------------------------------------------------------- GPU
BGS = {"black": (0.0, 0.0, 0.0), "white": (1.0, 1.0, 1.0), "rgb": (0.1, 0.2, 0.3)}
MASKS = ["zeros", "ones", "random30", "spatial20", "culled"]


def _golden(name):
    path = glob.glob(os.path.join(HERE, "golden", name + "*.npz"))[0]
    z = np.load(path)
    cloud = synth.Cloud(z["means3D"], z["scales"], z["rotations"], z["opacities"], z["shs"], int(z["sh_degree"]))
    cam = synth.Camera(int(z["H"]), int(z["W"]), float(z["tanfovx"]), float(z["tanfovy"]), z["viewmatrix"],
                       z["projmatrix"], z["campos"])
    cp = z["colors_precomp"] if z["colors_precomp"].size else None
    return cloud, cam, cp


def _scene(name):
    """(cloud, camera, colors_precomp or None)."""
    if name in ("c1", "c2", "c3", "hotspot"):
        return _golden({"c1": "c1_", "c2": "c2_", "c3": "c3_", "hotspot": "hotspot_"}[name])
    if name == "c3_20k":   # enough instances (R > 4096) for a speculative miss
        cloud, _ = synth.make_config("c3", P=20_000)
        return cloud, synth.ring_cameras(8, 4.5, 15.0, 320, 240, 61.0)[0], None
    if name == "needle":
        cloud, cam = synth.needle_cloud(P=600)
        return cloud, cam, None
    if name == "odd_frame":
        cloud, _ = synth.make_config("c3", P=8_000)
        return cloud, synth.ring_cameras(8, 4.5, 15.0, 333, 201, 61.0)[1], None
    cam = synth._origin_camera(48, 40)
    if name == "p1":
        xyz = synth._at_pixels(cam, np.array([20.0]), np.array([17.0]), np.array([3.0])).astype(np.float32)
        return synth.Cloud(xyz, np.full((1, 3), 0.08, np.float32), np.array([[1, 0, 0, 0]], np.float32),
                           np.array([[0.8]], np.float32), np.full((1, 1, 3), 0.3, np.float32), 0), cam, None
    if name == "p0":
        z = np.zeros((0, 3), np.float32)
        return synth.Cloud(z, z, np.zeros((0, 4), np.float32), np.zeros((0, 1), np.float32),
                           np.zeros((0, 1, 3), np.float32), 0), cam, None
    raise ValueError(name)


def _mask(kind, cloud, cam):
    P = cloud.means3D.shape[0]
    rng = np.random.default_rng(5)
    if kind == "zeros":
        m = np.zeros(P, bool)
    elif kind == "ones":
        m = np.ones(P, bool)
    elif kind == "random30":
        m = rng.uniform(size=P) < 0.3
    elif kind == "spatial20":   # GaussianEditor's typical edit: the 20 % nearest the origin
        d = np.linalg.norm(cloud.means3D, axis=1)
        m = d <= np.quantile(d, 0.2) if P else np.zeros(0, bool)
    elif kind == "culled":   # only Gaussians that the camera culls
        m = _plain(cloud, cam, (0, 0, 0), None)[0][1].cpu().numpy() == 0
    else:
        raise ValueError(kind)
    return torch.from_numpy(m).cuda()


def _inputs(cloud, cp):
    ct = cloud_tensors(cloud, "cuda")
    kw = dict(means3D=ct["means3D"], means2D=torch.zeros_like(ct["means3D"]), opacities=ct["opacities"],
              scales=ct["scales"], rotations=ct["rotations"])
    if cp is not None:
        kw["colors_precomp"] = torch.from_numpy(cp).cuda()
    else:
        kw["shs"] = ct["shs"]
    return kw


def _plain(cloud, cam, bg, cp, colors=None, **opt):
    """One forward through GaussianRasterizer (no gradients); `colors` replaces the colour input (forward #2)."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    rs = settings_from(cam, bg, cloud.sh_degree, "cuda", debug=opt.pop("debug", False))
    kw = _inputs(cloud, cp)
    if colors is not None:
        kw.pop("shs", None)
        kw["colors_precomp"] = colors
    rast = GaussianRasterizer(rs, **opt)
    with torch.no_grad():
        return rast(**kw), rast


def _second_forward(cloud, cam, bg, mask, activated=None):
    """GaussianEditor's forward #2: the mask as the colour of all three channels. `activated` = (opacities, scales,
    rotations) replaces the cloud's own (the PyTorch activations of the raw parameters)."""
    if activated is not None:
        op, sc, ro = (t.detach().cpu().numpy() for t in activated)
        cloud = synth.Cloud(cloud.means3D, sc, ro, op, cloud.shs, cloud.sh_degree)
    out, _ = _plain(cloud, cam, bg, None, colors=mask.float()[:, None].repeat(1, 3))
    return out[0]


def _activated(cloud):
    """sigmoid / exp / normalize of the raw parameters _run gives forward_raw, in PyTorch (the plain path's inputs)."""
    ct = cloud_tensors(cloud, "cuda")
    logit = torch.logit(ct["opacities"].clamp(1e-4, 1 - 1e-4))
    return (torch.sigmoid(logit), torch.exp(torch.log(ct["scales"])),
            torch.nn.functional.normalize(ct["rotations"].clone()))


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _key(cloud, cam):
    return (torch.cuda.current_device(), cloud.means3D.shape[0], cam.image_width, cam.image_height)


def _fused(cloud, cam, bg, cp, mask, form):
    """Forward #1 with mask_render in one forward form -> (outputs, rasterizer)."""
    import gaussianeditor_b200.rasterizer as RZ
    key = _key(cloud, cam)
    opt = {}
    if form == "exact":
        RZ._r_hint.pop(key, None)
    elif form == "hit":
        _plain(cloud, cam, bg, cp)   # leaves the hint
    elif form == "miss":
        RZ._r_hint[key] = 1          # capacity 4097
    elif form in ("static", "static_over"):
        _plain(cloud, cam, bg, cp)
        R = int(RZ._RasterizeGaussians.last_state.num_rendered)
        if form == "static_over" and R < 2:
            pytest.skip("R < 2: no overflowing capacity")
        opt["static_capacity"] = max(R, 1) if form == "static" else R - 1
    elif form == "debug":
        opt["debug"] = True
    spec = dict(RZ.SPEC_STATS)
    out, rast = _plain(cloud, cam, bg, cp, mask_render=mask, **opt)
    torch.cuda.synchronize()
    if form == "hit" and cloud.means3D.shape[0] > 0:
        assert RZ.SPEC_STATS["launched"] == spec["launched"] + 1 and RZ.SPEC_STATS["missed"] == spec["missed"]
    if form == "miss":
        assert RZ.SPEC_STATS["missed"] == spec["missed"] + 1
    return out, rast


SCENES = ["c1", "c2", "c3", "hotspot", "needle", "odd_frame", "p1", "p0", "c3_20k"]
FORMS = ["exact", "hit", "miss", "static", "static_over", "debug"]


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("scene", SCENES)
def test_mask_render_bit_identical_to_the_second_forward(scene, form):
    cloud, cam, cp = _scene(scene)
    P = cloud.means3D.shape[0]
    if form == "miss" and scene != "c3_20k":
        pytest.skip("a speculative miss needs more than 4096 instances")
    if form.startswith("static") and P == 0:
        pytest.skip("an empty cloud has no capacity to fill")
    H, W = cam.image_height, cam.image_width
    for kind in MASKS if P > 1 else ["zeros", "ones"]:
        mask = _mask(kind, cloud, cam)
        if kind == "culled" and not bool(mask.any()):
            continue
        for bgn, bg in BGS.items():
            out, rast = _fused(cloud, cam, bg, cp, mask, form)
            mimg = out[-1]
            assert len(out) == 4 and mimg.shape == (3, H, W) and mimg.dtype == torch.float32
            assert not mimg.requires_grad
            if form == "static_over":   # an empty frame: both images are the background
                assert int(rast.status[1]) == 1
                bgt = torch.tensor(bg, device="cuda")[:, None, None].expand(3, H, W)
                assert torch.equal(_bits(mimg), _bits(bgt.contiguous())), (kind, bgn)
                assert torch.equal(_bits(out[0]), _bits(bgt.contiguous())), (kind, bgn)
                continue
            ref = _second_forward(cloud, cam, bg, mask)
            assert torch.equal(_bits(mimg), _bits(ref)), (kind, bgn, (mimg != ref).sum().item())
            if P == 0:
                assert bool((_bits(mimg) == 0).all())


@pytest.mark.gpu
def test_uint8_mask_equals_bool_mask():
    cloud, cam, cp = _scene("c3")
    m = _mask("random30", cloud, cam)
    a, _ = _plain(cloud, cam, (0.1, 0.2, 0.3), cp, mask_render=m)
    b, _ = _plain(cloud, cam, (0.1, 0.2, 0.3), cp, mask_render=m.to(torch.uint8) * 9)
    assert torch.equal(_bits(a[-1]), _bits(b[-1]))


@pytest.mark.gpu
def test_constructor_validation_gpu():
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    cloud, cam, _ = _scene("c3")
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
    P = cloud.means3D.shape[0]
    with pytest.raises(ValueError, match="mask_render must be contiguous"):
        GaussianRasterizer(rs, mask_render=torch.ones(2 * P, dtype=torch.bool, device="cuda")[::2])
    m = torch.ones(P, dtype=torch.bool, device="cuda")
    r = GaussianRasterizer(rs, camera_grad=True, mask_render=m)   # unlike grad_mask, combinable with camera_grad
    assert r.mask_render.dtype == torch.uint8 and r.mask_render.data_ptr() == m.data_ptr()
    r = GaussianRasterizer(rs, mask_render=m[:-1])
    with pytest.raises(ValueError, match="mask_render has"):
        r(**_inputs(cloud, None))


# ---- nothing else moves ------------------------------------------------------------------------------------------------
MODES = ["sh", "colors", "depth", "alpha", "camera", "grad_mask", "raw", "static", "static_raw", "grad_mask_raw"]


def _run(cloud, cam, mode, mask_render=None, bg=(0.1, 0.2, 0.3), capacity=None, seed=0):
    """Deterministic forward + backward of one mode -> (forward outputs, gradients, forward state views); the forward
    outputs include "mask_render" when it is asked for."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians, forward_state_views
    dev = "cuda"
    ct = cloud_tensors(cloud, dev, requires_grad=True)
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    H, W = cam.image_height, cam.image_width
    g = torch.Generator(device=dev).manual_seed(seed)
    up_c, up_d, up_a = (torch.rand(c, H, W, generator=g, device=dev) for c in (3, 1, 1))
    edit = torch.from_numpy(np.random.default_rng(seed).uniform(size=cloud.means3D.shape[0]) < 0.4).cuda()
    means2D = torch.zeros_like(ct["means3D"], requires_grad=True)
    opt = dict(deterministic=True, return_alpha=mode == "alpha", depth_grad=mode == "depth")
    if mode == "camera":
        for k in ("viewmatrix", "projmatrix", "campos"):
            getattr(rs, k).requires_grad_(True)
        opt["camera_grad"] = True
    if mode.startswith("grad_mask"):
        opt["grad_mask"] = edit
    if capacity is not None:
        opt["static_capacity"] = capacity
    if mask_render is not None:
        opt["mask_render"] = mask_render
    rast = GaussianRasterizer(rs, **opt)
    leaves = {"means2D": means2D, "means3D": ct["means3D"]}
    if "raw" in mode:
        shs = ct["shs"].detach()
        dc = shs[:, :1].clone().requires_grad_(True)
        rest = shs[:, 1:].clone().requires_grad_(True)
        logit = torch.logit(ct["opacities"].detach().clamp(1e-4, 1 - 1e-4)).requires_grad_(True)
        lsc = torch.log(ct["scales"].detach()).requires_grad_(True)
        rot = ct["rotations"].detach().clone().requires_grad_(True)
        out = rast.forward_raw(ct["means3D"], means2D, logit, dc, rest, lsc, rot)
        leaves.update(dc=dc, rest=rest, logit=logit, lsc=lsc, rot=rot)
    else:
        kw = dict(means3D=ct["means3D"], means2D=means2D, opacities=ct["opacities"], scales=ct["scales"],
                  rotations=ct["rotations"])
        leaves.update(opacities=ct["opacities"], scales=ct["scales"], rotations=ct["rotations"])
        if mode == "colors":
            cp = torch.from_numpy(np.random.default_rng(seed).uniform(size=(cloud.means3D.shape[0], 3))
                                  .astype(np.float32)).cuda().requires_grad_(True)
            kw["colors_precomp"] = cp
            leaves["colors"] = cp
        else:
            kw["shs"] = ct["shs"]
            leaves["shs"] = ct["shs"]
        out = rast(**kw)
    if mode == "camera":
        leaves.update(view=rs.viewmatrix, proj=rs.projmatrix, campos=rs.campos)
    state = _RasterizeGaussians.last_state
    loss = (out[0] * up_c).sum() + (out[2] * up_d).sum()
    if mode == "alpha":
        loss = loss + (out[3] * up_a).sum()
    loss.backward()
    names = ["color", "radii", "depth"] + (["alpha"] if mode == "alpha" else [])
    fwd = {n: out[i].detach().cpu() for i, n in enumerate(names)}
    if mask_render is not None:
        assert len(out) == len(names) + 1 and not out[-1].requires_grad
        fwd["mask_render"] = out[-1].cpu()
    views = forward_state_views(state) if state.num_rendered is not None else {}
    fwd.update({k: views[k].cpu() for k in ("final_T", "n_contrib") if k in views})
    grads = {k: v.grad.detach().cpu().clone() for k, v in leaves.items() if v.grad is not None}
    return fwd, grads, state


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("scene", ["c3", "odd_frame"])
def test_other_outputs_and_gradients_unchanged(scene, mode):
    cloud, cam, _ = _scene(scene)
    mask = _mask("spatial20", cloud, cam)
    cap = None
    if mode.startswith("static"):
        _plain(cloud, cam, (0.1, 0.2, 0.3), None)
        from gaussianeditor_b200.rasterizer import _RasterizeGaussians
        cap = int(_RasterizeGaussians.last_state.num_rendered) + 7
    mode_ = {"static": "sh", "static_raw": "raw"}.get(mode, mode)
    ref_f, ref_g, _ = _run(cloud, cam, mode_, capacity=cap)
    got_f, got_g, _ = _run(cloud, cam, mode_, mask_render=mask, capacity=cap)
    assert set(got_f) == set(ref_f) | {"mask_render"} and ref_g.keys() == got_g.keys()
    for k in ref_f:
        assert torch.equal(_bits(ref_f[k]), _bits(got_f[k])), k
    for k in ref_g:
        assert torch.equal(_bits(ref_g[k]), _bits(got_g[k])), k
    if "raw" not in mode:
        assert torch.equal(_bits(got_f["mask_render"]), _bits(_second_forward(cloud, cam, (0.1, 0.2, 0.3), mask).cpu()))


@pytest.mark.gpu
def test_raw_path_mask_render():
    """forward_raw: an all-zero mask gives bg * final_T exactly; otherwise the image matches the plain path's second
    forward to the rounding of the in-kernel sigmoid."""
    cloud, cam, _ = _scene("odd_frame")
    bg = (0.1, 0.2, 0.3)
    zf, _, _ = _run(cloud, cam, "raw", mask_render=_mask("zeros", cloud, cam), bg=bg)
    want = torch.tensor(bg)[:, None, None] * zf["final_T"][None]
    assert torch.equal(_bits(zf["mask_render"]), _bits(want))
    for kind in ("spatial20", "random30", "ones"):
        mask = _mask(kind, cloud, cam)
        f, _, _ = _run(cloud, cam, "raw", mask_render=mask, bg=bg)
        ref = _second_forward(cloud, cam, bg, mask, _activated(cloud)).cpu()
        assert rel_l2(f["mask_render"].numpy(), ref.numpy()) <= 1e-5, kind
        assert float((f["mask_render"] - ref).abs().max()) <= 1e-4, kind


@pytest.mark.gpu
def test_not_differentiable_and_gradients_unchanged_by_a_loss_on_it():
    cloud, cam, _ = _scene("c3")
    mask = _mask("random30", cloud, cam)
    ref_f, ref_g, _ = _run(cloud, cam, "depth")
    got_f, got_g, _ = _run(cloud, cam, "depth", mask_render=mask)
    for k in ref_g:
        assert torch.equal(_bits(ref_g[k]), _bits(got_g[k])), k


@pytest.mark.gpu
@pytest.mark.parametrize("raw", [False, True])
def test_captured_step_replays_to_the_eager_bits(raw):
    """A static-capacity forward + backward with mask_render, captured in a CUDA graph, replays to the eager step's
    bits (all outputs, the mask image and every gradient)."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    cloud, cam, _ = _scene("odd_frame")
    mask = _mask("spatial20", cloud, cam)
    rs = settings_from(cam, (0.1, 0.2, 0.3), cloud.sh_degree, "cuda")
    _plain(cloud, cam, (0.1, 0.2, 0.3), None)
    from gaussianeditor_b200.rasterizer import _RasterizeGaussians
    cap = int(_RasterizeGaussians.last_state.num_rendered) * 2 + 64
    rast = GaussianRasterizer(rs, static_capacity=cap, deterministic=True, grad_mask=mask, mask_render=mask)
    ct = cloud_tensors(cloud, "cuda", requires_grad=True)
    params = [ct["means3D"], ct["opacities"], ct["scales"], ct["rotations"], ct["shs"]]
    if raw:
        params = [ct["means3D"], torch.logit(ct["opacities"].detach().clamp(1e-4, 1 - 1e-4)).requires_grad_(True),
                  torch.log(ct["scales"].detach()).requires_grad_(True),
                  ct["rotations"].detach().clone().requires_grad_(True),
                  ct["shs"].detach()[:, :1].clone().requires_grad_(True),
                  ct["shs"].detach()[:, 1:].clone().requires_grad_(True)]
    means2D = torch.zeros_like(ct["means3D"], requires_grad=True)
    up = torch.rand(3, cam.image_height, cam.image_width, device="cuda", generator=torch.Generator("cuda").manual_seed(1))

    def step():
        for p in params + [means2D]:
            p.grad = None
        if raw:
            m3, lo, ls, ro, dc, rest = params
            out = rast.forward_raw(m3, means2D, lo, dc, rest, ls, ro)
        else:
            m3, op, sc, ro, sh = params
            out = rast(means3D=m3, means2D=means2D, opacities=op, shs=sh, scales=sc, rotations=ro)
        (out[0] * up).sum().backward()
        return [out[0].detach(), out[2].detach(), out[-1]] + [p.grad for p in params + [means2D]]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = [t.clone() for t in step()]
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    for t in captured:
        t.fill_(-1.0)
    graph.replay()
    torch.cuda.synchronize()
    assert int(rast.status[1]) == 0
    for i, (a, b) in enumerate(zip(eager, captured)):
        assert torch.equal(_bits(a), _bits(b)), i
    if not raw:   # the raw image matches the second forward to the sigmoid's rounding only (test_raw_path_mask_render)
        assert torch.equal(_bits(captured[2]), _bits(_second_forward(cloud, cam, (0.1, 0.2, 0.3), mask)))


@pytest.mark.gpu
def test_render_returns_mask_render():
    from gaussianeditor_b200 import edit_loop, gaussian_renderer as GR
    from types import SimpleNamespace
    cloud, cams = synth.make_config("c5", P=3_000)
    scene = edit_loop.EditScene(cloud, "cuda")
    view = edit_loop.make_view(cams[0], "cuda")
    pipe = SimpleNamespace(convert_SHs_python=False, compute_cov3D_python=False, debug=False)
    bg = torch.zeros(3, device="cuda")
    pkg = GR.render(view, scene, pipe, bg, grad_mask=scene.mask, mask_render=scene.mask)
    sem = GR.render(view, scene, pipe, bg, override_color=scene.mask[..., None].float().repeat(1, 3))["render"]
    assert torch.equal(_bits(pkg["mask_render"]), _bits(sem))
    assert "mask_render" not in GR.render(view, scene, pipe, bg)


# ---- harness -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cuda_graph", [False, True])
def test_edit_loop_fused_semantic_equals_second_forward(cuda_graph):
    from gaussianeditor_b200 import edit_loop
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    runs = {}
    for sem in ("render", "fused"):
        log = []
        runs[sem] = (edit_loop.run_edit_loop(GaussianRasterizer, steps=12, P=6_000, densification_interval=6, seed=3,
                                             deterministic=True, grad_mask="kernel", cuda_graph=cuda_graph,
                                             semantic=sem, semantic_log=log), log)
    (a, la), (b, lb) = runs["render"], runs["fused"]
    assert a["losses"] == b["losses"] and a["counts"] == b["counts"]
    assert torch.equal(a["max_radii2D"], b["max_radii2D"])
    for k in a["params"]:
        assert torch.equal(_bits(a["params"][k]), _bits(b["params"][k])), k
    assert len(la) == len(lb) == 12
    for i, (x, y) in enumerate(zip(la, lb)):
        assert torch.equal(x, y), i
    assert any(bool(x.any()) for x in la)


def test_edit_loop_rejects_an_unknown_semantic_source():
    from gaussianeditor_b200 import edit_loop
    with pytest.raises(ValueError, match="semantic"):
        edit_loop.run_edit_loop(None, steps=1, semantic="twice")
