"""Fixed-capacity forward (`GaussianRasterizer(static_capacity=...)`, gsr_forward_static / gsr_forward_static_raw).

CPU: the entry points are declared, exported and bound; bad arguments are rejected before anything touches a device;
`static_capacity` with `debug=True` raises ValueError before any launch; `render` passes the option only when given.
GPU: against the default (host-sized) path on the parity cases and at config-3 size, for plain and raw inputs with
alpha / depth / camera outputs: images, radii and alpha are the same bits, status = {R, 0}, deterministic gradients
are the same bits (so the forward state the backward reads is the same) and the others within 1e-6 relative L2, or
within four times the default path's own call-to-call spread where its float atomics spread further. The rotation
gradients, small sums of cancelling terms, get 1e-5: at 1M Gaussians the two paths' float atomics put them a few 1e-6
apart while two default calls were 6e-7 apart. A captured forward + backward replayed for three cameras
equals eager calls bit for bit. At capacity R/2, on both binning paths, the frame is empty (background, zero depth and
alpha), every backward returns exact zeros and `check_capacity()` raises. The edit loop gives the same Gaussian counts
and losses with and without CUDA-graph replay.
"""
import contextlib
import ctypes as C
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import _lib, gaussian_renderer as GR, synth
from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians
from util import rel_l2, settings_from

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, WORKSPACE = -1, -3  # GSR_ERR_INVALID, GSR_ERR_WORKSPACE
NAMES = ("gsr_forward_static", "gsr_forward_static_raw")
D = C.c_void_p(256)          # a 16-byte aligned fake device pointer: nothing may dereference it
BIG = 1 << 30


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_entry_points_are_declared_exported_and_bound():
    header = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    lib = _lib.load()
    for name in NAMES:
        assert re.search(r"GSR_API int " + name + r"\(", header), name
        assert name in _lib.SYMBOLS
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == 14


def _err(rc, want, text):
    assert rc == want, (rc, _lib.load().gsr_last_error())
    assert text.encode() in _lib.load().gsr_last_error(), _lib.load().gsr_last_error()


def _settings(W=64, H=48, M=16, deg=3):
    return _lib.Settings(H, W, 1.0, 1.0, 1.0, deg, M, 0, 0, D, D, D, D)


def _call(raw=False, s=None, cloud=None, cap=100, geom=D, gbytes=BIG, binning=D, bbytes=BIG, image=D, ibytes=BIG,
          radii=D, color=D, depth=D, status=D):
    lib = _lib.load()
    s = _settings() if s is None else s
    if raw:
        cloud = _lib.RawCloud(100, D, D, D, D, D, D) if cloud is None else cloud
        fn = lib.gsr_forward_static_raw
    else:
        cloud = _lib.Cloud(100, D, D, D, None, D, D, None) if cloud is None else cloud
        fn = lib.gsr_forward_static
    return fn(C.byref(s), C.byref(cloud), cap, geom, gbytes, binning, bbytes, image, ibytes, radii, color, depth,
              status, None)


@pytest.mark.parametrize("raw", [False, True])
def test_forward_static_validates_before_touching_the_device(raw):
    for cap in (0, -5):
        _err(_call(raw, cap=cap), INVALID, "static capacity must be positive")
    _err(_call(raw, status=None), INVALID, "status is null")
    _err(_call(raw, color=None), INVALID, "output images are null")
    _err(_call(raw, depth=None), INVALID, "output images are null")
    _err(_call(raw, radii=None), INVALID, "radii / geometry workspace is null")
    _err(_call(raw, geom=None), INVALID, "radii / geometry workspace is null")
    _err(_call(raw, s=_settings(deg=3, M=9)), INVALID, "sh_degree")
    if raw:
        _err(_call(raw, cloud=_lib.RawCloud(100, None, D, D, D, D, D)), INVALID, "must not be null")
        _err(_call(raw, cloud=_lib.RawCloud(100, D, D, D, None, D, D)), INVALID, "features_rest is null")
        _err(_call(raw, cloud=_lib.RawCloud(100, D, D, D, C.c_void_p(260), D, D)), INVALID, "16-byte aligned")
    else:
        _err(_call(raw, cloud=_lib.Cloud(100, None, D, D, None, D, D, None)), INVALID, "must not be null")
        _err(_call(raw, cloud=_lib.Cloud(100, D, D, D, D, D, D, None)), INVALID, "one of either SHs")
        _err(_call(raw, cloud=_lib.Cloud(-1, D, D, D, None, D, D, None)), INVALID, "negative size")


def _cpu_settings(debug):
    z = torch.zeros
    return GR.GaussianRasterizationSettings(48, 64, 1.0, 1.0, z(3), 1.0, torch.eye(4), torch.eye(4), 0, z(3), False,
                                            debug)


def test_static_capacity_with_debug_raises_before_any_launch():
    rast = GaussianRasterizer(_cpu_settings(True), static_capacity=1000)
    x = torch.zeros(10, 3)
    with pytest.raises(ValueError, match="debug"):
        rast(x, x, torch.zeros(10, 1), shs=torch.zeros(10, 1, 3), scales=x, rotations=torch.zeros(10, 4))
    with pytest.raises(ValueError, match="debug"):
        rast.forward_raw(x, x, torch.zeros(10, 1), torch.zeros(10, 1, 3), torch.zeros(10, 0, 3), x,
                         torch.zeros(10, 4))
    assert rast.status is None
    for bad in (0, -1, 2.5, True, 2 ** 31):
        with pytest.raises(ValueError, match="static_capacity"):
            GaussianRasterizer(_cpu_settings(False), static_capacity=bad)
    with pytest.raises(RuntimeError, match="check_capacity"):
        GaussianRasterizer(_cpu_settings(False), static_capacity=10).check_capacity()


def test_render_passes_static_capacity_only_when_given(monkeypatch):
    seen = []

    class Recorder:
        def __init__(self, raster_settings, **kw):
            seen.append(kw)
            self.status = torch.tensor([7, 0], dtype=torch.int32)

        def __call__(self, means3D, **kw):
            P = means3D.shape[0]
            return torch.zeros(3, 4, 4), torch.ones(P, dtype=torch.int32), torch.zeros(1, 4, 4)

    monkeypatch.setattr(GR, "GaussianRasterizer", Recorder)
    pc = SimpleNamespace(get_xyz=torch.zeros(5, 3), get_opacity=torch.ones(5, 1), get_scaling=torch.ones(5, 3),
                         get_rotation=torch.ones(5, 4), get_features=torch.zeros(5, 1, 3), active_sh_degree=0)
    cam = SimpleNamespace(image_height=4, image_width=4, FoVx=1.0, FoVy=1.0, world_view_transform=torch.eye(4),
                          full_proj_transform=torch.eye(4), camera_center=torch.zeros(3))
    pipe = SimpleNamespace(convert_SHs_python=False, compute_cov3D_python=False)
    out = GR.render(cam, pc, pipe, torch.zeros(3))
    assert seen[-1] == {} and "status" not in out
    out = GR.render(cam, pc, pipe, torch.zeros(3), static_capacity=123)
    assert seen[-1] == {"static_capacity": 123}
    assert out["status"].tolist() == [7, 0]
    GR.render(cam, pc, pipe, torch.zeros(3), static_capacity=9, deterministic=True, depth_grad=True)
    assert seen[-1] == {"static_capacity": 9, "deterministic": True, "depth_grad": True}


# ---------------------------------------------------------------------------------------------------------------- GPU
@contextlib.contextmanager
def _option(name, value):
    old = _lib.load().gsr_get_option(name.encode())
    _lib.set_option(name, value)
    try:
        yield
    finally:
        _lib.set_option(name, old)


def _cases(full=True):
    c1, cams1 = synth.make_config("c1")
    c3, _ = synth.make_config("c3", P=60_000)
    cam3 = synth.ring_cameras(8, 4.5, 15.0, 400, 304, 61.0)[2]
    cam_odd = synth.ring_cameras(8, 4.5, 15.0, 333, 201, 61.0)[5]
    out = [("c1", c1, cams1[0], (0.0, 0.0, 0.0)), ("c3s", c3, cam3, (1.0, 1.0, 1.0)),
           ("c3odd", c3, cam_odd, (0.2, 0.5, 0.7))]
    if full:
        c3f, cams3f = synth.make_config("c3")
        out.append(("c3full", c3f, cams3f[0], (0.0, 0.0, 0.0)))
    return out


def _inputs(cloud, raw, dev):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    P = cloud.means3D.shape[0]
    m2 = torch.zeros(P, 3, device=dev)
    if raw:
        op = t(cloud.opacities).clamp(1e-6, 1 - 1e-6)
        xs = [t(cloud.means3D), m2, torch.log(op / (1 - op)), t(cloud.shs[:, :1]).contiguous(),
              t(cloud.shs[:, 1:]).contiguous(), torch.log(t(cloud.scales)), t(cloud.rotations) * 2.0]
    else:
        xs = [t(cloud.means3D), m2, t(cloud.opacities), t(cloud.shs), t(cloud.scales), t(cloud.rotations)]
    return [x.detach().clone().requires_grad_(True) for x in xs]


def _run(rs, cloud, raw, flags, det, cap, dev, up):
    """One forward + backward; returns (outputs, grads, module)."""
    alpha, depth, camera = ("alpha" in flags), ("depth" in flags), ("camera" in flags)
    if camera:
        rs = rs._replace(viewmatrix=rs.viewmatrix.detach().clone().requires_grad_(True),
                         projmatrix=rs.projmatrix.detach().clone().requires_grad_(True),
                         campos=rs.campos.detach().clone().requires_grad_(True))
    rast = GaussianRasterizer(rs, return_alpha=alpha, camera_grad=camera, depth_grad=depth, deterministic=det,
                              static_capacity=cap)
    xs = _inputs(cloud, raw, dev)
    if raw:
        outs = rast.forward_raw(*xs)
    else:
        outs = rast(xs[0], xs[1], xs[2], shs=xs[3], scales=xs[4], rotations=xs[5])
    loss = (outs[0] * up["color"]).sum()
    if depth:
        loss = loss + (outs[2] * up["depth"]).sum()
    if alpha:
        loss = loss + (outs[3] * up["alpha"]).sum()
    loss.backward()
    grads = [x.grad for x in xs]
    if camera:
        grads += [rs.viewmatrix.grad, rs.projmatrix.grad, rs.campos.grad]
    return [o.detach() for o in outs], grads, rast


def _upstream(cam, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    H, W = cam.image_height, cam.image_width
    return dict(color=torch.rand(3, H, W, generator=g, device=dev), depth=torch.rand(1, H, W, generator=g, device=dev),
                alpha=torch.rand(1, H, W, generator=g, device=dev))


ROT = {False: 5, True: 6}   # index of the rotation gradient in _run's list (plain, raw)
COMBOS = [(False, ()), (False, ("alpha",)), (False, ("depth",)), (False, ("camera",)),
          (False, ("alpha", "depth", "camera")), (True, ()), (True, ("depth",))]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["c1", "c3s", "c3odd", "c3full"])
def test_static_equals_default_path(case):
    dev = torch.device("cuda")
    name, cloud, cam, bg = [c for c in _cases(full=case == "c3full") if c[0] == case][0]
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    up = _upstream(cam, dev)
    for raw, flags in COMBOS:
        for det in (True, False):
            ref_out, ref_g, _ = _run(rs, cloud, raw, flags, det, None, dev, up)
            R = _RasterizeGaussians.last_state.num_rendered
            if not det:   # the float atomics' call-to-call spread of the default path itself, over two repeats
                spread = [0.0] * len(ref_g)
                for _ in range(2):
                    again = _run(rs, cloud, raw, flags, det, None, dev, up)[1]
                    spread = [max(sp, rel_l2(a.cpu().numpy(), b.cpu().numpy()))
                              for sp, a, b in zip(spread, again, ref_g)]
            for cap in (R, int(R * 1.25) + 4096):
                out, g, rast = _run(rs, cloud, raw, flags, det, cap, dev, up)
                tag = (case, raw, flags, det, cap)
                assert rast.status.tolist() == [R, 0], tag
                assert rast.check_capacity() == R
                for a, b in zip(out, ref_out):
                    assert torch.equal(a, b), tag
                for k, (a, b) in enumerate(zip(g, ref_g)):
                    if det:
                        assert torch.equal(a, b), tag
                    else:
                        e = rel_l2(a.cpu().numpy(), b.cpu().numpy())
                        assert e <= max(1e-6, 4 * spread[k], 1e-5 if k == ROT[raw] else 0.0), (tag, k, e, spread[k])


@pytest.mark.gpu
def test_captured_forward_backward_replays_bit_exact():
    dev = torch.device("cuda")
    cloud, _ = synth.make_config("c3", P=60_000)
    cams = synth.ring_cameras(8, 4.5, 15.0, 400, 304, 61.0)
    rs0 = settings_from(cams[0], (0.1, 0.2, 0.3), cloud.sh_degree, dev)
    up = _upstream(cams[0], dev)
    caps = []
    for cam in cams[:3]:   # a capacity that holds for every replayed camera
        _run(settings_from(cam, (0.1, 0.2, 0.3), cloud.sh_degree, dev), cloud, False, (), True, None, dev, up)
        caps.append(_RasterizeGaussians.last_state.num_rendered)
    cap = int(max(caps) * 1.25) + 4096
    # static camera tensors the graph reads; intrinsics are shared
    rs = rs0._replace(viewmatrix=rs0.viewmatrix.clone(), projmatrix=rs0.projmatrix.clone(), campos=rs0.campos.clone())
    rast = GaussianRasterizer(rs, return_alpha=True, depth_grad=True, deterministic=True, static_capacity=cap)
    xs = _inputs(cloud, False, dev)

    def step():
        for x in xs:
            x.grad = None
        col, radii, depth, alpha = rast(xs[0], xs[1], xs[2], shs=xs[3], scales=xs[4], rotations=xs[5])
        ((col * up["color"]).sum() + (depth * up["depth"]).sum() + (alpha * up["alpha"]).sum()).backward()
        return [col, radii, depth, alpha] + [x.grad for x in xs]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
        status = rast.status
    for i, cam in enumerate(cams[:3]):
        rsi = settings_from(cam, (0.1, 0.2, 0.3), cloud.sh_degree, dev)
        rs.viewmatrix.copy_(rsi.viewmatrix); rs.projmatrix.copy_(rsi.projmatrix); rs.campos.copy_(rsi.campos)
        graph.replay()
        got = [t.clone() for t in captured]
        st = status.tolist()
        eager = GaussianRasterizer(rsi, return_alpha=True, depth_grad=True, deterministic=True, static_capacity=cap)
        ex = _inputs(cloud, False, dev)
        col, radii, depth, alpha = eager(ex[0], ex[1], ex[2], shs=ex[3], scales=ex[4], rotations=ex[5])
        ((col * up["color"]).sum() + (depth * up["depth"]).sum() + (alpha * up["alpha"]).sum()).backward()
        want = [col.detach(), radii, depth.detach(), alpha.detach()] + [x.grad for x in ex]
        assert st == [caps[i], 0] and eager.status.tolist() == st
        for k, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), (i, k)


@pytest.mark.gpu
@pytest.mark.parametrize("binning_variant", [1, 0])
def test_overflow_renders_an_empty_frame_with_zero_gradients(binning_variant):
    dev = torch.device("cuda")
    name, cloud, cam, bg = _cases(full=False)[2]
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    up = _upstream(cam, dev)
    H, W = cam.image_height, cam.image_width
    with _option("binning_variant", binning_variant):
        _run(rs, cloud, False, (), True, None, dev, up)
        R = _RasterizeGaussians.last_state.num_rendered
        cap = R // 2
        bgimg = torch.tensor(bg, dtype=torch.float32, device=dev)[:, None, None].expand(3, H, W)
        for raw, flags in COMBOS:
            for det in (True, False):
                out, grads, rast = _run(rs, cloud, raw, flags, det, cap, dev, up)
                tag = (binning_variant, raw, flags, det)
                assert rast.status.tolist() == [R, 1], tag
                assert torch.equal(out[0], bgimg), tag
                assert int(torch.count_nonzero(out[2])) == 0, tag
                if "alpha" in flags:
                    assert int(torch.count_nonzero(out[3])) == 0, tag
                for g in grads:
                    assert int(torch.count_nonzero(g)) == 0, tag
                with pytest.raises(RuntimeError, match=f"R={R} exceeds static_capacity={cap}"):
                    rast.check_capacity()
    assert _lib.load().gsr_get_option(b"binning_variant") == 1


@pytest.mark.gpu
def test_forward_static_checks_workspace_sizes_before_any_launch():
    lib = _lib.load()
    s = _settings(W=64, H=48)
    P, cap = 100, 1000
    gb, bb, ib = lib.gsr_geometry_bytes(P), lib.gsr_binning_bytes(P, cap, 64, 48), lib.gsr_image_bytes(64, 48)
    for raw in (False, True):
        _err(_call(raw, s=s, cap=cap, gbytes=gb - 1, bbytes=bb, ibytes=ib), WORKSPACE, "geometry workspace too small")
        _err(_call(raw, s=s, cap=cap, gbytes=gb, bbytes=bb - 1, ibytes=ib), WORKSPACE, "binning workspace too small")
        _err(_call(raw, s=s, cap=cap, gbytes=gb, bbytes=bb, binning=None, ibytes=ib), WORKSPACE,
             "binning workspace too small")
        _err(_call(raw, s=s, cap=cap, gbytes=gb, bbytes=bb, ibytes=ib - 1), WORKSPACE, "image workspace too small")


@pytest.mark.gpu
def test_empty_cloud_writes_zero_status_and_images():
    dev = torch.device("cuda")
    cam = synth.ring_cameras(8, 4.5, 15.0, 64, 48, 61.0)[0]
    rs = settings_from(cam, (0.5, 0.5, 0.5), 0, dev)
    rast = GaussianRasterizer(rs, static_capacity=10)
    rast.status = torch.full((2,), 9, dtype=torch.int32, device=dev)
    e = torch.zeros(0, 3, device=dev)
    col, radii, depth = rast(e, e, torch.zeros(0, 1, device=dev), shs=torch.zeros(0, 1, 3, device=dev), scales=e,
                             rotations=torch.zeros(0, 4, device=dev))
    assert rast.status.tolist() == [0, 0] and radii.numel() == 0
    assert int(torch.count_nonzero(col)) == 0 and int(torch.count_nonzero(depth)) == 0


@pytest.mark.gpu
def test_edit_loop_graph_replay_equals_eager_steps():
    from gaussianeditor_b200.edit_loop import run_edit_loop
    kw = dict(steps=100, P=20_000, densification_interval=30, deterministic=True)
    eager = run_edit_loop(GaussianRasterizer, static_capacity=True, **kw)
    graph = run_edit_loop(GaussianRasterizer, cuda_graph=True, **kw)
    assert eager["counts"] == graph["counts"]
    assert len(graph["capacities"]) == 4           # three densifications: four Gaussian counts, four graphs
    assert eager["losses"] == graph["losses"]
    assert eager["capacities"] == graph["capacities"]
    assert torch.equal(eager["max_radii2D"], graph["max_radii2D"])
