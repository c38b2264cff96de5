"""Alpha image and camera-pose gradients on the Gaussian-sharded rasterizer (return_alpha, camera_grad).

CPU: the new entry points are declared, exported and bound and reject bad arguments before touching a device;
forward_raw refuses both flags before any collective; combine_camera_rows over gloo gives every rank the numpy
rank-ordered fp32 sum bit for bit; the kernels of the deterministic camera path have no float atomics.
GPU: `world` virtual ranks on one GPU drive the step functions (dense with shared geometry, sparse through
SS.link_virtual, with the camera partials travelling through gsr_peer_row_put). The alpha frame equals the single-GPU
alpha; per-Gaussian gradients of colour + alpha, alpha-only and colour + alpha + depth losses match the single-GPU
backward within the sharded tolerance; the camera gradients of the whole cloud are the same bits on every virtual rank
and match GaussianRasterizer(camera_grad=True). Deterministic mode repeats its bits, dense equals sparse, and at world 1
everything equals the single-GPU deterministic call. With both flags off the launches per step and the peer block are
unchanged. The module runs under torchrun through tools/sharded_check.py --alpha --camera-grad.
"""
import ctypes as C
import os
import re
import shutil
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from gaussianeditor_b200 import _lib, sharded as S
from util import rel_l2
from test_sharded_fused_depth import (_OneRank, _act_inputs, _bits_equal, _case, _named,
                                      _rank_args, _upstreams)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gaussianeditor_b200", "csrc", "libgsr_b200.so")
INVALID, WORKSPACE = -1, -3  # GSR_ERR_INVALID, GSR_ERR_WORKSPACE
NEW_NAMES = ("gsr_shard_alpha_image", "gsr_shard_backward_render_alpha", "gsr_shard_backward_preprocess_camera",
             "gsr_sparse_backward_preprocess_camera", "gsr_frame_broadcast_planes", "gsr_peer_row_put")
CAM = ("viewmatrix", "projmatrix", "campos")


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_new_entry_points_are_declared_exported_and_bound():
    header = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    lib = _lib.load()
    assert lib.gsr_abi_version() == 2
    for name in NEW_NAMES:
        assert re.search(r"GSR_API int " + name + r"\(", header), name
        assert name in _lib.SYMBOLS
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and fn.argtypes is not None
    assert "no alpha or camera gradient" not in header


D = C.c_void_p(256)          # a 16-byte aligned fake device pointer: nothing may dereference it
BIG = 1 << 30


def _settings(M=16, deg=3):
    return _lib.Settings(64, 64, 1.0, 1.0, 1.0, deg, M, 0, 0, D, D, D, D)


def _err(rc, want, text):
    assert rc == want, (rc, _lib.load().gsr_last_error())
    assert text.encode() in _lib.load().gsr_last_error(), _lib.load().gsr_last_error()


def test_shard_alpha_image_validates_before_touching_the_device():
    lib = _lib.load()
    need = lib.gsr_image_bytes(64, 48)

    def call(owner=_lib.TileOwner(2, 1), image=D, ibytes=need, W=64, H=48, out=D):
        return lib.gsr_shard_alpha_image(None if owner is None else C.byref(owner), image, ibytes, W, H, out, None)
    _err(call(owner=None), INVALID, "row_stride")
    for stride, phase in [(2, 2), (0, 0), (3, -1)]:
        _err(call(owner=_lib.TileOwner(stride, phase)), INVALID, "row_stride")
    _err(call(image=None), INVALID, "bad arguments")
    _err(call(out=None), INVALID, "bad arguments")
    _err(call(W=-1), INVALID, "bad arguments")
    _err(call(ibytes=need - 1), WORKSPACE, "image workspace too small")


def test_shard_backward_render_alpha_validates_before_touching_the_device():
    lib = _lib.load()
    s = _settings()
    P, R = 100, 10
    need = lib.gsr_deterministic_scratch_bytes(P, R, 0)

    def call(owner=_lib.TileOwner(2, 1), P=P, R=R, alpha=D, depth=None, det=None, dbytes=0, acc_bytes=1 << 20):
        return lib.gsr_shard_backward_render_alpha(C.byref(s), C.byref(owner), P, R, D, 1 << 20, D, 1 << 20, D,
                                                   1 << 20, D, alpha, depth, D, acc_bytes, det, dbytes, None)
    _err(call(alpha=None), INVALID, "dL_dout_alpha is null")
    _err(call(alpha=None, depth=D), INVALID, "dL_dout_alpha is null")
    for stride, phase in [(2, 2), (0, 0), (3, -1)]:
        _err(call(owner=_lib.TileOwner(stride, phase)), INVALID, "row_stride")
    _err(call(R=-1), INVALID, "bad arguments")
    _err(call(P=0), INVALID, "bad arguments")
    _err(call(acc_bytes=P * 12 * 4 - 4), WORKSPACE, "accumulators too small")
    _err(call(det=D, dbytes=need - 1), WORKSPACE, "deterministic scratch")
    _err(call(depth=D, det=D, dbytes=need - 1), WORKSPACE, "deterministic scratch")


def test_preprocess_camera_entry_points_validate_before_touching_the_device():
    lib = _lib.load()
    s = _settings()
    P = 100
    cloud = _lib.Cloud(P, D, D, D, None, D, D, None)
    grads = _lib.Grads(D, D, D, D, D, D, D, D)
    cneed = lib.gsr_camera_scratch_bytes(P)
    good = _lib.CameraGrads(D, D, D, D, cneed)

    def dense(cam=good, base=100, P_total=300):
        return lib.gsr_shard_backward_preprocess_camera(C.byref(s), C.byref(cloud), P_total, base, D, BIG, D, D,
                                                        C.byref(grads), 1, None if cam is None else C.byref(cam), None)

    def sparse(cam=good, plan=_lib.SparsePlan(3, 1, 100, 64), acc_bytes=BIG):
        return lib.gsr_sparse_backward_preprocess_camera(C.byref(s), C.byref(cloud), C.byref(plan), D, BIG, D, D, BIG,
                                                         D, acc_bytes, C.byref(grads), 0,
                                                         None if cam is None else C.byref(cam), None)
    for call in (dense, sparse):
        _err(call(cam=None), INVALID, "camera gradients: null struct")
        _err(call(cam=_lib.CameraGrads(None, D, D, D, cneed)), INVALID, "null struct or output")
        _err(call(cam=_lib.CameraGrads(D, D, None, D, cneed)), INVALID, "null struct or output")
        _err(call(cam=_lib.CameraGrads(D, D, D, D, cneed - 1)), WORKSPACE, "camera scratch too small")
        _err(call(cam=_lib.CameraGrads(D, D, D, None, cneed)), WORKSPACE, "camera scratch too small")
    _err(dense(base=250), INVALID, "does not fit")
    _err(sparse(plan=_lib.SparsePlan(3, 3, 100, 64)), INVALID, "sparse plan")
    _err(sparse(plan=_lib.SparsePlan(3, 1, 99, 64)), INVALID, "does not fit slice_len")
    _err(sparse(acc_bytes=P * 48 - 4), WORKSPACE, "acc_slice too small")


def test_frame_broadcast_planes_and_row_put_validate_before_touching_the_device():
    lib = _lib.load()
    peers = (C.c_void_p * 3)(D, D, D)

    def planes(n=5, owner=_lib.TileOwner(3, 1), frame=D, ptrs=peers):
        return lib.gsr_frame_broadcast_planes(C.byref(owner), 64, 48, n, frame, ptrs, None)
    for n in (0, -1, 6):
        _err(planes(n), INVALID, "planes")
    _err(planes(owner=_lib.TileOwner(3, 3)), INVALID, "frame_broadcast: bad arguments")
    _err(planes(owner=_lib.TileOwner(9, 1)), INVALID, "frame_broadcast: bad arguments")
    _err(planes(frame=None), INVALID, "frame_broadcast: bad arguments")
    _err(planes(ptrs=(C.c_void_p * 3)(D, None, D)), INVALID, "peer frame 1 is null")

    def put(world=3, rank=1, row=D, n=35, ptrs=peers):
        return lib.gsr_peer_row_put(world, rank, row, n, ptrs, None)
    for n in (0, 65):
        _err(put(n=n), INVALID, "peer_row_put: n")
    _err(put(world=0, rank=0), INVALID, "peer_row_put: bad arguments")
    _err(put(world=9), INVALID, "peer_row_put: bad arguments")
    _err(put(rank=3), INVALID, "peer_row_put: bad arguments")
    _err(put(row=None), INVALID, "peer_row_put: bad arguments")
    _err(put(ptrs=(C.c_void_p * 3)(D, D, None)), INVALID, "peer slots 2 are null")


class _NoCollective:
    """An exchange whose every collective fails the test: the calls below must raise before reaching one."""
    world, rank = 2, 0

    def __getattr__(self, name):
        raise AssertionError(f"collective {name} reached")


def _module(rs, P, mode="dense", pool=None, exchange=None, **flags):
    """ShardedGaussianRasterizer of a one-rank group (or with `exchange`), built without torch.distributed."""
    m = S.ShardedGaussianRasterizer.__new__(S.ShardedGaussianRasterizer)
    nn.Module.__init__(m)
    m.raster_settings = rs
    m.deterministic, m.depth_grad = bool(flags.get("deterministic")), bool(flags.get("depth_grad"))
    m.return_alpha, m.camera_grad = bool(flags.get("return_alpha")), bool(flags.get("camera_grad"))
    m.exchange = exchange or _OneRank()
    m.plan, m.mode = S.ShardPlan(P, m.exchange.world, m.exchange.rank), mode
    m.pool, m.sparse_pool = None, pool
    return m


@pytest.mark.parametrize("flags", [dict(return_alpha=True), dict(camera_grad=True),
                                   dict(return_alpha=True, camera_grad=True, depth_grad=True)])
def test_forward_raw_refuses_alpha_and_camera_before_any_collective(flags):
    P = 10
    raw = (torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 1), torch.zeros(P, 1, 3), torch.zeros(P, 15, 3),
           torch.zeros(P, 3), torch.ones(P, 4))
    for mode in ("dense", "sparse"):
        m = _module(None, 2 * P, mode=mode, exchange=_NoCollective(), **flags)
        with pytest.raises(ValueError, match="forward_raw is not available on a module built with") as e:
            m.forward_raw(*raw)
        for f in ("return_alpha", "camera_grad"):
            assert (f + "=True" in str(e.value)) == bool(flags.get(f))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rows(world):
    """Every rank's camera partial (rank 1's is a zero row, as from a rank without Gaussians)."""
    g = np.random.default_rng(17)
    rows = (g.standard_normal((world, S.CAM_ROW)) * 10.0 ** g.integers(-3, 4, (world, S.CAM_ROW))).astype(np.float32)
    rows[1] = 0
    return rows


def _combine_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ex = S.Exchange()
        rows = torch.full((world, S.CAM_ROW), float("nan"))
        rows[rank] = torch.from_numpy(_rows(world)[rank])
        ex.all_gather_inplace(rows)
        out[rank] = S.combine_camera_rows(rows).numpy().tobytes()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_combine_camera_rows_over_gloo_gives_every_rank_the_rank_ordered_sum(world):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_combine_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    rows = _rows(world)
    want = rows[0].copy()
    for r in range(1, world):
        want = (want + rows[r]).astype(np.float32)   # fp32 adds in ascending rank order
    assert all(out[r] == want.tobytes() for r in range(world))


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="cuobjdump is not available")
def test_alpha_and_camera_kernels_have_no_float_atomics():
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
    # the new owner alpha and row-put kernels, the CAM (and CAM+DEPTH) preprocess backward and the camera reduction
    cam_bwd = re.compile(r"preprocess_bwd_kernelILb[01]ELb0ELb1ELb[01]EE")
    picked = {n: b for n, b in kernels.items()
              if any(k in n for k in ("alpha_image_owner_kernel", "peer_row_put_kernel", "camera_reduce_kernel"))
              or cam_bwd.search(n)}
    assert len(picked) == 7, sorted(picked)
    fatom = re.compile(r"^(?:@!?U?P\w+\s+)?(RED|ATOM)[GS]?\.\S*\.F(16|32|64)")
    for n, body in picked.items():
        assert body and not [i for i in body if fatom.match(i)], n


# ---------------------------------------------------------------------------------------------------------------- GPU
def _cam_settings(rs):
    return rs._replace(**{k: getattr(rs, k).clone().requires_grad_(True) for k in CAM})


def _alpha_upstream(size, seed):
    g = torch.Generator().manual_seed(1000 + seed)
    W, H = size
    return (torch.rand(1, H, W, generator=g) - 0.5).cuda()


def _ups(loss, dL, dA, dD):
    """(colour, alpha or None, depth or None) upstream gradients of a loss, as autograd hands them to the backward."""
    return (dL if "color" in loss else torch.zeros_like(dL), dA if "alpha" in loss else None,
            dD if "depth" in loss else None)


def _loss(loss, out, dL, dA, dD):
    total = 0.0
    if "color" in loss:
        total = total + (out[0] * dL).sum()
    if "alpha" in loss:
        total = total + (out[3] * dA).sum()
    if "depth" in loss:
        total = total + (out[2] * dD).sum()
    return total


def _single(rs, d, loss=None, ups=None, det=False):
    """GaussianRasterizer(return_alpha, camera_grad, depth_grad): (colour, depth, alpha), radii, gradients by name,
    camera gradients by name."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    rs = _cam_settings(rs)
    r = GaussianRasterizer(rs, return_alpha=True, camera_grad=True, depth_grad=True, deterministic=det)
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in d.items()}
    m2 = torch.zeros_like(d["means3D"], requires_grad=True)
    out = r(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], shs=leaves["shs"],
            scales=leaves["scales"], rotations=leaves["rotations"])
    g = cams = None
    if loss is not None:
        _loss(loss, out, *ups).backward()
        g = {k: v.grad for k, v in leaves.items()}
        g["means2D"] = m2.grad
        cams = {k: getattr(rs, k).grad.clone() for k in CAM}
    return (out[0].detach(), out[2].detach(), out[3].detach()), out[1], g, cams


def _cams_of(total, rs):
    return dict(zip(CAM, S.camera_grads_like(total, rs)))


def _dense(world, rs, d, loss=None, ups=None, det=False):
    """Virtual dense ranks: (colour, depth, alpha), radii of the real Gaussians, gradients by name, camera gradients
    by name as every rank computes them (one dict per rank)."""
    P = d["means3D"].shape[0]
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    geom = radii = None
    bufs = []
    for p in plans:
        args, _ = _rank_args(d, p)
        b = S.shard_preprocess(p, rs, *args, geom=geom, radii=radii)
        geom, radii = b.geom, b.radii
        bufs.append(b)
    for b in bufs:
        b.geom = geom.clone(); b.radii = torch.full_like(radii, -7)
    frames, accs = [], []
    for b in bufs:
        S.shard_order(b)
        frame = torch.zeros(5, rs.image_height, rs.image_width, device="cuda")
        S.shard_render(b, frame[:3], frame[3:4])
        S.shard_alpha(b, frame[4:])
        frames.append(frame)
        if loss is not None:
            gc, ga, gd = _ups(loss, *ups)
            accs.append(S.shard_backward_render(b, gc, det, gd, ga).clone())
    frame = torch.stack(frames).sum(0)
    radii_real = torch.cat([S.shard_slice(b.radii, b.plan) for b in bufs])
    grads = cams = None
    if loss is not None:
        acc = accs[0].clone()
        for a in accs[1:]:
            acc += a   # ascending rank order, what reduce_scatter_ordered does
        per, rows = [], []
        for b in bufs:
            row, cam = S.camera_row(b.plan.count, "cuda")
            per.append(S.shard_backward_preprocess(b, acc[b.plan.base:b.plan.base + b.plan.slice_len].contiguous(),
                                                   "depth" in loss, cam))
            rows.append(row)
        grads = _named(per, False)
        gathered = torch.stack(rows)   # what the all-gather leaves on every rank
        cams = [_cams_of(S.combine_camera_rows(gathered.clone()), rs) for _ in bufs]
    return (frame[:3], frame[3:4], frame[4:]), radii_real, grads, cams


def _sparse(world, rs, d, cap_mode, loss=None, ups=None, det=False):
    from gaussianeditor_b200 import sparse_sharded as SS
    P = d["means3D"].shape[0]
    ranks = [SS.SparseRank(S.ShardPlan(P, world, r), torch.device("cuda"), rs.image_width, rs.image_height,
                           alpha=True, camera=True) for r in range(world)]
    SS.link_virtual(ranks)

    def order(cap):
        for rk in ranks:
            rk.matrix.zero_()
        steps = []
        for rk in ranks:
            args, _ = _rank_args(d, rk.plan)
            steps.append(SS.sparse_preprocess(rk, rs, *args, cap))
        m = torch.stack([rk.matrix for rk in ranks]).sum(0)
        for rk in ranks:
            rk.matrix.copy_(m)
        return steps, [SS.sparse_order(st) for st in steps]
    cap0 = ranks[0].cap_alloc
    steps, res = order(cap0)
    maxc = res[0][1]
    if cap_mode == "tight":
        steps, res = order(max(maxc, 1))
    elif cap_mode == "overflow" and maxc > 1:
        steps, res = order(max(1, maxc // 2))
        assert all(r[1] > st.cap for r, st in zip(res, steps))
        steps, res = order(SS.next_capacity(maxc, cap0))
    assert all(r[1] <= st.cap for r, st in zip(res, steps))
    for rk in ranks:
        rk.frame.fill_(float("nan"))   # the sparse frame is not zero-filled: every pixel needs its one writer
    for st in steps:
        SS.sparse_render(st, st.rk.frame[:3], st.rk.frame[3:4])
        SS.sparse_alpha(st, st.rk.frame[4:5])
    for rk in ranks:
        SS.frame_broadcast(rk)
    frame = ranks[0].frame.clone()
    assert all(torch.equal(rk.frame, frame) for rk in ranks[1:])
    radii_real = torch.cat([rk.radii_local[:rk.plan.count] for rk in ranks])
    grads = cams = None
    if loss is not None:
        gc, ga, gd = _ups(loss, *ups)
        accs = [SS.sparse_backward_render(st, gc, det, gd, ga) for st in steps]
        for st, acc in zip(steps, accs):
            SS.sparse_return(st, acc)
        for rk in ranks:
            rk.cam_slots.fill_(float("nan"))
        per = []
        for st in steps:
            row, cam = S.camera_row(st.n, "cuda")
            per.append(SS.sparse_backward_preprocess(st, "depth" in loss, cam))
            SS.camera_put(st.rk, row)
        grads = _named(per, False)
        cams = [_cams_of(S.combine_camera_rows(rk.cam_slots[:, :S.CAM_ROW]), rs) for rk in ranks]
    return (frame[:3], frame[3:4], frame[4:5]), radii_real, grads, cams


FWD_CASES = [  # world, (W, H), SH degree, sparse capacity
    (1, (400, 300), 3, "full"),
    (2, (333, 201), 3, "tight"),
    (3, (333, 201), 0, "overflow"),
    (8, (400, 300), 0, "tight"),
    (8, (64, 40), 3, "overflow"),        # 3 tile rows: five ranks own none
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,size,deg,cap_mode", FWD_CASES)
def test_alpha_frame_bit_identical_to_single_gpu(world, size, deg, cap_mode):
    rs, t = _case(size, deg)
    d = _act_inputs(t, 16)
    (color, depth, alpha), radii, _, _ = _single(rs, d)
    assert int((radii > 0).sum()) > 1000 and float(alpha.max()) > 0.5
    for mode in ("dense", "sparse"):
        (c, dp, a), r, _, _ = _dense(world, rs, d) if mode == "dense" else _sparse(world, rs, d, cap_mode)
        assert torch.equal(a, alpha), mode
        assert torch.equal(c, color) and torch.equal(dp, depth), mode
        assert torch.equal(r, radii), mode


BWD_WORLDS = [(2, (333, 201), 3, "tight"), (3, (400, 300), 3, "overflow"), (8, (64, 40), 0, "full")]


@pytest.mark.gpu
@pytest.mark.parametrize("world,size,deg,cap_mode", BWD_WORLDS)
@pytest.mark.parametrize("loss", ["color+alpha", "alpha", "color+alpha+depth"])
def test_gaussian_gradients_with_alpha_match_single_gpu(loss, world, size, deg, cap_mode):
    rs, t = _case(size, deg)
    d = _act_inputs(t, 16)
    dL, dD = _upstreams(size, world)
    ups = (dL, _alpha_upstream(size, world), dD)
    _, _, ref, _ = _single(rs, d, loss, ups)
    for mode in ("dense", "sparse"):
        g = (_dense(world, rs, d, loss, ups) if mode == "dense" else _sparse(world, rs, d, cap_mode, loss, ups))[2]
        assert g.keys() == ref.keys(), mode
        for k in ref:
            assert rel_l2(g[k].cpu().numpy(), ref[k].cpu().numpy()) <= 2e-5, (mode, k)
    if loss == "color+alpha":   # the alpha term really moves the gradients
        _, _, no_alpha, _ = _single(rs, d, "color", ups)
        assert rel_l2(ref["opacities"].cpu().numpy(), no_alpha["opacities"].cpu().numpy()) > 1e-3


CAM_WORLDS = [(1, (400, 300), 3, "full"), (3, (333, 201), 3, "overflow"), (8, (64, 40), 0, "tight")]


@pytest.mark.gpu
@pytest.mark.parametrize("world,size,deg,cap_mode", CAM_WORLDS)
@pytest.mark.parametrize("loss", ["color", "color+depth", "color+alpha+depth"])
def test_camera_gradients_match_single_gpu_and_agree_on_every_rank(loss, world, size, deg, cap_mode):
    rs, t = _case(size, deg)
    d = _act_inputs(t, 16)
    dL, dD = _upstreams(size, 20 + world)
    ups = (dL, _alpha_upstream(size, 20 + world), dD)
    _, _, _, ref = _single(rs, d, loss, ups)
    _, _, _, ref2 = _single(rs, d, loss, ups)
    spread = max(rel_l2(ref2[k].cpu().numpy(), ref[k].cpu().numpy()) for k in CAM)
    bound = max(1e-4, 10 * spread)
    worst = 0.0
    for mode in ("dense", "sparse"):
        cams = (_dense(world, rs, d, loss, ups) if mode == "dense" else _sparse(world, rs, d, cap_mode, loss, ups))[3]
        assert len(cams) == world
        for other in cams[1:]:
            _bits_equal(other, cams[0])                 # the same bits on every rank
        c = cams[0]
        assert not c["viewmatrix"][:, 3].any() and not c["projmatrix"][:, 2].any(), mode   # entries never read
        for k in CAM:
            e = rel_l2(c[k].cpu().numpy(), ref[k].cpu().numpy())
            worst = max(worst, e)
            assert e <= bound, (mode, k, e, spread)
    print(f"camera rel L2: world={world} loss={loss} worst={worst:.2e} single-GPU spread={spread:.2e}")


DET_WORLDS = [(1, (400, 300), 3, ("full", "tight")), (3, (333, 201), 3, ("tight", "overflow")),
              (8, (64, 40), 0, ("overflow", "full"))]


@pytest.mark.gpu
@pytest.mark.parametrize("world,size,deg,caps", DET_WORLDS)
def test_deterministic_alpha_camera_repeatable_dense_equals_sparse(world, size, deg, caps):
    loss = "color+alpha+depth"
    rs, t = _case(size, deg)
    d = _act_inputs(t, 16)
    dL, dD = _upstreams(size, 30 + world)
    ups = (dL, _alpha_upstream(size, 30 + world), dD)
    _, _, dense, dcam = _dense(world, rs, d, loss, ups, det=True)
    _, _, again, acam = _dense(world, rs, d, loss, ups, det=True)
    _bits_equal(dense, again)
    _bits_equal(dcam[0], acam[0])
    _, _, sparse, scam = _sparse(world, rs, d, caps[0], loss, ups, det=True)
    _, _, sparse2, scam2 = _sparse(world, rs, d, caps[1], loss, ups, det=True)
    _bits_equal(sparse, sparse2)
    _bits_equal(scam[0], scam2[0])
    _bits_equal(dense, sparse)
    _bits_equal(dcam[0], scam[0])
    if world == 1:
        _, _, ref, rcam = _single(rs, d, loss, ups, det=True)
        _bits_equal(dense, ref)
        _bits_equal(dcam[0], rcam)


def _module_step(m, rs, d, loss, ups):
    """One forward + backward through the module: outputs, gradients by name, camera gradients by name."""
    rs = _cam_settings(rs) if m.camera_grad else rs
    m.raster_settings = rs
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in d.items()}
    m2 = torch.zeros_like(d["means3D"], requires_grad=True)
    out = m(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], shs=leaves["shs"],
            scales=leaves["scales"], rotations=leaves["rotations"])
    _loss(loss, out, *ups).backward()
    g = {k: v.grad for k, v in leaves.items()}
    g["means2D"] = m2.grad
    cams = {k: getattr(rs, k).grad for k in CAM} if m.camera_grad else {}
    return [o.detach() for o in out], g, cams


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["dense", "sparse"])
def test_module_at_one_rank_equals_single_gpu_and_unused_alpha_changes_nothing(mode):
    """The autograd functions through the module (a one-rank group, deterministic): every loss gives
    GaussianRasterizer(deterministic, return_alpha, camera_grad, depth_grad)'s bits, camera arrays included; an alpha
    output without a loss gives the bits of return_alpha=False; the flags-off step launches what it launched before
    this feature, and each flag adds exactly its own kernels."""
    size = (333, 201)
    rs, t = _case(size, 3)
    d = _act_inputs(t, 16)
    P = d["means3D"].shape[0]
    dL, dD = _upstreams(size, 5)
    ups = (dL, _alpha_upstream(size, 5), dD)
    flags = dict(deterministic=True, return_alpha=True, camera_grad=True, depth_grad=True)

    def pool(alpha, camera):   # a one-rank SparsePool without a process group
        if mode == "dense":
            return None
        from gaussianeditor_b200 import sparse_sharded as SS
        rk = SS.SparseRank(S.ShardPlan(P, 1, 0), torch.device("cuda"), *size, alpha=alpha, camera=camera)
        SS.link_virtual([rk])
        p = SS.SparsePool.__new__(SS.SparsePool)
        p.all, p.free, p.cap, p.redo = [rk], [rk], rk.cap_alloc, 0
        return p
    m = _module(rs, P, mode=mode, pool=pool(True, True), **flags)
    for loss in ("color+alpha+depth", "alpha", "color", "depth"):
        out, g, cams = _module_step(m, rs, d, loss, ups)
        (c, dp, a), r, rg, rcam = _single(rs, d, loss, ups, det=True)
        assert torch.equal(out[0], c) and torch.equal(out[2], dp) and torch.equal(out[3], a) and torch.equal(out[1], r)
        _bits_equal(g, rg)
        _bits_equal(cams, rcam)
    off = _module(rs, P, mode=mode, pool=pool(False, False), deterministic=True)
    alpha_only = _module(rs, P, mode=mode, pool=pool(True, False), deterministic=True, return_alpha=True)
    _bits_equal(_module_step(alpha_only, rs, d, "color", ups)[1], _module_step(off, rs, d, "color", ups)[1])

    def launches(mod, loss):
        _module_step(mod, rs, d, loss, ups)   # warm: the caching allocator and the sparse capacity settle
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        _module_step(mod, rs, d, loss, ups)
        torch.cuda.synchronize()
        return _lib.launch_count() - n0
    base = launches(off, "color")
    assert launches(alpha_only, "color") == base + 1                    # the owner alpha kernel
    cam_only = _module(rs, P, mode=mode, pool=pool(False, True), deterministic=True, camera_grad=True)
    extra = 1 if mode == "dense" else 3    # camera_reduce_kernel; sparse: + the row put and its barrier
    assert launches(cam_only, "color") == base + extra


@pytest.mark.gpu
def test_flags_off_peer_block_keeps_its_size_and_layout():
    from gaussianeditor_b200 import sparse_sharded as SS
    lib = _lib.load()
    for world, (W, H) in ((1, (333, 201)), (3, (400, 300)), (8, (64, 40))):
        plan = S.ShardPlan(60013, world, world - 1)
        rk = SS.SparseRank(plan, torch.device("cuda"), W, H)
        want = SS.CTRL_BYTES + SS._align(16 * W * H)   # [control words | 4-plane frame | candidates]
        assert rk.frame_off == SS.CTRL_BYTES and rk.frame_bytes == want and rk.planes == 4
        assert rk.total_bytes == want + lib.gsr_sparse_candidate_bytes(world, max(plan.slice_len, 1))
        with pytest.raises(RuntimeError, match="without camera slots"):
            rk.cam_slots
        both = SS.SparseRank(plan, torch.device("cuda"), W, H, alpha=True, camera=True)
        assert both.cam_off == SS.CTRL_BYTES + SS._align(20 * W * H)
        assert both.frame_bytes == both.cam_off + SS.CAM_SLOT_BYTES
        rk.close(); both.close()


def _torchrun(variant, nproc):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    args = {"dense-nccl": [], "dense-p2p": ["--p2p"], "sparse": ["--mode", "sparse"]}[variant]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sharded_check.py"), "--config", "c3",
           "--P", "30001", "--alpha", "--camera-grad"] + args
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    child = "\n".join(l for l in r.stderr.splitlines() if l.startswith("[rank"))
    assert r.returncode == 0, r.stdout[-2000:] + child[-3000:] + r.stderr[-2000:]
    assert "SHARDED_CHECK_OK" in r.stdout and "alpha_camera=ok" in r.stdout, r.stdout[-2000:]
    print(r.stdout.strip().splitlines()[0])


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
@pytest.mark.parametrize("variant", ["dense-nccl", "dense-p2p", "sparse"])
def test_torchrun_sharded_check_alpha_camera_grad(variant, nproc):
    """return_alpha=True and camera_grad=True (with depth_grad) under torchrun, one process per GPU: frames bit-identical
    to one GPU, gradients within tolerance, camera gradients the same bits on every rank."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    _torchrun(variant, nproc)
