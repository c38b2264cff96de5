"""Fused activations (forward_raw) and the depth gradient (depth_grad) on the Gaussian-sharded rasterizer.

CPU: the new entry points are declared, exported and bound, and reject null, misaligned and out-of-range arguments
before touching a device; ShardedGaussianRasterizer.forward_raw and depth_grad check their arguments like their
single-GPU counterparts.
GPU: `world` virtual ranks on one GPU drive the step functions (dense with shared geometry, sparse through
SS.link_virtual). RAW frames, depth and radii are bit-identical to GaussianRasterizer.forward_raw; the dense peer-store
RAW preprocess writes the same record bytes into every peer as the plain RAW preprocess; gradients of RAW, activated +
depth and RAW + depth match the single-GPU backward within the sharded tolerance, and in deterministic mode they repeat
their bits, dense equals sparse, and at world 1 they are the single-GPU deterministic bits. The autograd functions give
depth_grad's semantics (a depth-only loss works; a colour-only loss gives the depth_grad=False bits). The module runs
under torchrun through tools/sharded_check.py --raw --depth-grad.
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

from gaussianeditor_b200 import _lib, sharded as S, synth
from util import cloud_tensors, rel_l2, settings_from

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, WORKSPACE = -1, -3  # GSR_ERR_INVALID, GSR_ERR_WORKSPACE
NEW_NAMES = ("gsr_shard_preprocess_raw", "gsr_shard_preprocess_p2p_raw", "gsr_sparse_preprocess_raw",
             "gsr_shard_backward_render_depth", "gsr_shard_backward_preprocess_depth",
             "gsr_sparse_backward_preprocess_depth", "gsr_shard_backward_preprocess_raw",
             "gsr_sparse_backward_preprocess_raw")


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


D = C.c_void_p(256)          # a 16-byte aligned fake device pointer: nothing may dereference it
MIS = C.c_void_p(260)        # misaligned
BIG = 1 << 30                # a workspace size that passes every size check


def _settings(M=16, deg=3):
    return _lib.Settings(64, 64, 1.0, 1.0, 1.0, deg, M, 0, 0, D, D, D, D)


def _raw_cloud(P=100, rest=D, rot=D):
    return _lib.RawCloud(P, D, D, D, rest, D, rot)


def _raw_grads(rest=D, rot=D, m2=D):
    return _lib.RawGrads(D, m2, D, D, rest, D, rot)


def _grads(rot=D, m3=D):
    return _lib.Grads(m3, D, D, D, D, D, D, rot)


def _cloud(P=100):
    return _lib.Cloud(P, D, D, D, None, D, D, None)


def _err(rc, want, text):
    assert rc == want, (rc, _lib.load().gsr_last_error())
    assert text.encode() in _lib.load().gsr_last_error(), _lib.load().gsr_last_error()


def test_shard_preprocess_raw_entry_points_validate_before_touching_the_device():
    lib = _lib.load()
    s = _settings()

    def dense(rc=None, P_total=300, base=100, slice_len=100, geom=D, radii=D, gbytes=1 << 30):
        return lib.gsr_shard_preprocess_raw(C.byref(s), None if rc is None else C.byref(rc), P_total, base, slice_len,
                                            geom, gbytes, radii, None)
    _err(dense(), INVALID, "null settings/cloud")
    _err(dense(_raw_cloud(rest=MIS)), INVALID, "features_rest must be 16-byte aligned")
    _err(dense(_raw_cloud(rest=None)), INVALID, "features_rest is null")
    _err(dense(_raw_cloud(rot=MIS)), INVALID, "rotations must be 16-byte aligned")
    _err(dense(_raw_cloud(), base=250), INVALID, "does not fit")
    _err(dense(_raw_cloud(P=101)), INVALID, "does not fit")
    _err(dense(_raw_cloud(), radii=None), INVALID, "is null")

    peers = (C.c_void_p * 3)(D, D, D)

    def p2p(rc=None, world=3, rank=1, base=100, ptrs=peers, radii=D):
        return lib.gsr_shard_preprocess_p2p_raw(C.byref(s), None if rc is None else C.byref(rc), 300, base, 100, ptrs,
                                                world, rank, BIG, radii, None)
    _err(p2p(), INVALID, "null settings/cloud")
    _err(p2p(_raw_cloud(rest=MIS)), INVALID, "features_rest must be 16-byte aligned")
    _err(p2p(_raw_cloud(), world=9), INVALID, "p2p preprocess")
    _err(p2p(_raw_cloud(), rank=3), INVALID, "p2p preprocess")
    _err(p2p(_raw_cloud(), base=201), INVALID, "does not fit")
    _err(p2p(_raw_cloud(), radii=None), INVALID, "radii is null")


    def sparse(rc=None, plan=_lib.SparsePlan(3, 1, 100, 64), local=D, lbytes=1 << 30):
        return lib.gsr_sparse_preprocess_raw(C.byref(s), None if rc is None else C.byref(rc), C.byref(plan), local,
                                             lbytes, D, peers, BIG, D, None)
    _err(sparse(), INVALID, "does not fit slice_len")
    _err(sparse(_raw_cloud(rest=MIS)), INVALID, "features_rest must be 16-byte aligned")
    _err(sparse(_raw_cloud(P=101)), INVALID, "does not fit slice_len")
    _err(sparse(_raw_cloud(), plan=_lib.SparsePlan(0, 0, 100, 64)), INVALID, "sparse plan")
    _err(sparse(_raw_cloud(), plan=_lib.SparsePlan(3, 3, 100, 64)), INVALID, "sparse plan")
    _err(sparse(_raw_cloud(), local=None), INVALID, "null buffer")


def test_shard_backward_render_depth_validates_before_touching_the_device():
    lib = _lib.load()
    s = _settings()
    P, R = 100, 10
    need = lib.gsr_deterministic_scratch_bytes(P, R, 0)

    def call(owner=_lib.TileOwner(2, 1), P=P, R=R, depth=D, det=None, dbytes=0, acc_bytes=1 << 20):
        return lib.gsr_shard_backward_render_depth(C.byref(s), C.byref(owner), P, R, D, 1 << 20, D, 1 << 20, D,
                                                   1 << 20, D, depth, D, acc_bytes, det, dbytes, None)
    _err(call(depth=None), INVALID, "dL_dout_depth is null")
    for stride, phase in [(2, 2), (0, 0), (3, -1)]:
        _err(call(owner=_lib.TileOwner(stride, phase)), INVALID, "row_stride")
    _err(call(R=-1), INVALID, "bad arguments")
    _err(call(P=0), INVALID, "bad arguments")
    _err(call(acc_bytes=P * 48 - 1), WORKSPACE, "accumulators too small")
    _err(call(det=D, dbytes=need - 1), WORKSPACE, "deterministic scratch")


def test_shard_backward_preprocess_depth_and_raw_validate_before_touching_the_device():
    lib = _lib.load()
    s = _settings()

    def depth(c=_cloud(), gr=_grads(), base=100, acc=D):
        return lib.gsr_shard_backward_preprocess_depth(C.byref(s), C.byref(c), 300, base, D, BIG, D, acc,
                                                       None if gr is None else C.byref(gr), None)
    _err(depth(gr=None), INVALID, "grads / accumulators / radii is null")
    _err(depth(gr=_grads(m3=None)), INVALID, "a gradient output pointer is null")
    _err(depth(gr=_grads(rot=MIS)), INVALID, "dL_drotations must be 16-byte aligned")
    _err(depth(acc=MIS), INVALID, "acc_slice must be 16-byte aligned")
    _err(depth(base=201), INVALID, "does not fit P_total")

    def raw(rc=_raw_cloud(), gr=_raw_grads(), base=100, acc=D, flag=1):
        return lib.gsr_shard_backward_preprocess_raw(C.byref(s), None if rc is None else C.byref(rc), 300, base, D, BIG,
                                                     D, acc, None if gr is None else C.byref(gr), flag, None)
    _err(raw(rc=None), INVALID, "null settings/cloud")
    _err(raw(rc=_raw_cloud(rest=MIS)), INVALID, "features_rest must be 16-byte aligned")
    _err(raw(gr=None), INVALID, "grads / accumulators / radii is null")
    _err(raw(gr=_raw_grads(m2=None)), INVALID, "a gradient output pointer is null")
    _err(raw(gr=_raw_grads(rest=MIS)), INVALID, "16-byte aligned")
    _err(raw(gr=_raw_grads(rot=MIS), flag=0), INVALID, "16-byte aligned")
    _err(raw(acc=MIS), INVALID, "acc_slice must be 16-byte aligned")
    _err(raw(base=201), INVALID, "does not fit P_total")

    plan = _lib.SparsePlan(3, 1, 100, 64)

    def sdepth(c=_cloud(), gr=_grads(), acc=D, abytes=100 * 48, pl=plan):
        return lib.gsr_sparse_backward_preprocess_depth(C.byref(s), C.byref(c), C.byref(pl), D, BIG, D, D, BIG, acc,
                                                        abytes, None if gr is None else C.byref(gr), None)
    _err(sdepth(gr=None), INVALID, "null argument")
    _err(sdepth(gr=_grads(rot=MIS)), INVALID, "16-byte aligned")
    _err(sdepth(acc=MIS), INVALID, "16-byte aligned")
    _err(sdepth(c=_cloud(P=101)), INVALID, "does not fit slice_len")
    _err(sdepth(pl=_lib.SparsePlan(3, 1, 100, 0)), INVALID, "sparse plan")
    _err(sdepth(abytes=100 * 48 - 1), WORKSPACE, "acc_slice too small")

    def sraw(rc=_raw_cloud(), gr=_raw_grads(), acc=D, abytes=100 * 48):
        return lib.gsr_sparse_backward_preprocess_raw(C.byref(s), None if rc is None else C.byref(rc), C.byref(plan), D,
                                                      BIG, D, D, BIG, acc, abytes, None if gr is None else C.byref(gr), 1,
                                                      None)
    _err(sraw(rc=None), INVALID, "does not fit slice_len")
    _err(sraw(rc=_raw_cloud(rest=MIS)), INVALID, "features_rest must be 16-byte aligned")
    _err(sraw(gr=None), INVALID, "null argument")
    _err(sraw(gr=_raw_grads(rest=MIS)), INVALID, "16-byte aligned")
    _err(sraw(acc=MIS), INVALID, "acc_slice must be 16-byte aligned")
    _err(sraw(abytes=100 * 48 - 1), WORKSPACE, "acc_slice too small")


class _OneRank:
    """The collectives of a one-rank group (nothing to exchange): lets the autograd functions run without a process
    group."""
    world, rank = 1, 0

    def all_gather_inplace(self, total):
        pass

    def barrier(self, device):
        pass

    def all_reduce_sum(self, t):
        pass

    def reduce_scatter_sum(self, total, out):
        out.copy_(total[:out.shape[0]])

    reduce_scatter_ordered = reduce_scatter_sum


def _module(rs, P, deterministic=False, depth_grad=False, mode="dense", pool=None):
    """ShardedGaussianRasterizer of a one-rank group, built without torch.distributed."""
    m = S.ShardedGaussianRasterizer.__new__(S.ShardedGaussianRasterizer)
    nn.Module.__init__(m)
    m.raster_settings, m.deterministic, m.depth_grad = rs, bool(deterministic), bool(depth_grad)
    m.exchange, m.plan, m.mode = _OneRank(), S.ShardPlan(P, 1, 0), mode
    m.pool, m.sparse_pool = None, pool
    return m


def _cpu_settings():
    cam = synth.ring_cameras(8, 4.5, 15.0, 64, 48, 61.0)[0]
    return settings_from(cam, (0, 0, 0), 3, "cpu")


def test_forward_raw_and_depth_grad_check_their_arguments_like_the_single_gpu_path():
    rs = _cpu_settings()
    P = 10
    raw = (torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 1), torch.zeros(P, 1, 3), torch.zeros(P, 15, 3),
           torch.zeros(P, 3), torch.ones(P, 4))
    m = _module(rs, P, depth_grad=True)
    assert m.depth_grad is True and _module(rs, P, depth_grad=0).depth_grad is False
    with pytest.raises(RuntimeError, match="means3D must have dimensions"):
        m.forward_raw(torch.zeros(P, 4), *raw[1:])
    with pytest.raises(RuntimeError, match="needs CUDA tensors"):
        m.forward_raw(*raw)
    # torch's deterministic flag: the same rule as forward
    torch.use_deterministic_algorithms(True)
    try:
        with pytest.raises(RuntimeError, match="deterministic=True"):
            m.forward_raw(*raw)
        with pytest.raises(RuntimeError, match="needs CUDA tensors"):   # accepted; fails later on the CPU tensors
            _module(rs, P, deterministic=True, depth_grad=True).forward_raw(*raw)
        torch.use_deterministic_algorithms(True, warn_only=True)
        with pytest.warns(UserWarning, match="deterministic=True"), pytest.raises(RuntimeError, match="CUDA"):
            m.forward_raw(*raw)
    finally:
        torch.use_deterministic_algorithms(False)
    # the activated forward keeps its reference checks with depth_grad on
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        m(raw[0], raw[1], raw[2])
    with pytest.raises(Exception, match="exactly one of either scale/rotation pair"):
        m(raw[0], raw[1], raw[2], shs=torch.zeros(P, 16, 3))


# ---------------------------------------------------------------------------------------------------------------- GPU
_CLOUD = {}


def _full():
    if not _CLOUD:
        cloud, _ = synth.make_config("c3", P=60013)   # not divisible by the world sizes: padded tail on the last rank
        _CLOUD["cloud"] = cloud
        _CLOUD["t"] = cloud_tensors(cloud, "cuda")
    return _CLOUD["cloud"], _CLOUD["t"]


def _raw_inputs(t, M):
    """Raw parameters with M = 1 + K allocated coefficients (K = 0: features_rest [P, 0, 3])."""
    o = t["opacities"].clamp(1e-6, 1 - 1e-6)
    return dict(means3D=t["means3D"], opacity_logits=torch.log(o / (1 - o)),
                features_dc=t["shs"][:, :1].contiguous(), features_rest=t["shs"][:, 1:M].contiguous(),
                log_scales=torch.log(t["scales"]), raw_rotations=t["rotations"] * 1.7)


def _act_inputs(t, M):
    return dict(means3D=t["means3D"], shs=t["shs"][:, :M].contiguous(), opacities=t["opacities"],
                scales=t["scales"], rotations=t["rotations"])


RAW_ORDER = ("means3D", "means2D", "opacity_logits", "features_dc", "features_rest", "log_scales", "raw_rotations")
ACT_ORDER = ("means3D", "means2D", "shs", "colors", "opacities", "scales", "rotations", "cov")


def _rank_args(d, p):
    """(positional step-function inputs, raw_rest) of rank p."""
    sl = lambda k: S.shard_slice(d[k], p)
    empty = torch.empty(0, device="cuda")
    if "features_rest" in d:
        return (sl("means3D"), sl("features_dc"), empty, sl("opacity_logits"), sl("log_scales"), sl("raw_rotations"),
                empty), sl("features_rest")
    return (sl("means3D"), sl("shs"), empty, sl("opacities"), sl("scales"), sl("rotations"), empty), None


def _case(size, deg):
    _, t = _full()
    W, H = size
    cam = synth.ring_cameras(8, 4.5, 15.0, W, H, 61.0)[2]
    return settings_from(cam, (0.2, 0.5, 0.1), deg, "cuda"), t


def _single(rs, d, loss, dL, dD, depth_grad, det):
    """GaussianRasterizer (forward_raw for raw inputs): frames, radii and the gradients of every input + means2D."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in d.items()}
    m2 = torch.zeros_like(d["means3D"], requires_grad=True)
    r = GaussianRasterizer(rs, depth_grad=depth_grad, deterministic=det)
    if "features_rest" in d:
        color, radii, depth = r.forward_raw(leaves["means3D"], m2, leaves["opacity_logits"], leaves["features_dc"],
                                            leaves["features_rest"], leaves["log_scales"], leaves["raw_rotations"])
    else:
        color, radii, depth = r(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"],
                                shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"])
    if loss is not None:
        _loss(loss, color, depth, dL, dD).backward()
    g = {k: v.grad for k, v in leaves.items()}
    g["means2D"] = m2.grad
    return color.detach(), depth.detach(), radii, g


def _loss(loss, color, depth, dL, dD):
    return {"color": (color * dL).sum(), "both": (color * dL).sum() + (depth * dD).sum(),
            "depth": (depth * dD).sum()}[loss]


def _named(per_rank, raw):
    order = RAW_ORDER if raw else ACT_ORDER
    out = {}
    for i, name in enumerate(order):
        if name in ("colors", "cov"):
            continue
        out[name] = torch.cat([g[i] for g in per_rank])
    return out


def _upstream(loss, dL, dD):
    """(colour gradient, depth gradient or None) of a loss, as autograd hands them to the backward."""
    color = dL if loss != "depth" else torch.zeros_like(dL)
    return color, (dD if loss != "color" else None)


def _dense(world, rs, d, loss=None, dL=None, dD=None, det=False):
    """Virtual dense ranks: (colour, depth, radii of the real Gaussians, gradients by name or None)."""
    P = d["means3D"].shape[0]
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    geom = radii = None
    bufs = []
    for p in plans:
        args, rest = _rank_args(d, p)
        b = S.shard_preprocess(p, rs, *args, geom=geom, radii=radii, raw_rest=rest)
        geom, radii = b.geom, b.radii
        bufs.append(b)
    for b in bufs:
        b.geom = geom.clone(); b.radii = torch.full_like(radii, -7)
    frames, accs = [], []
    for b in bufs:
        S.shard_order(b)
        frame = torch.zeros(4, rs.image_height, rs.image_width, device="cuda")
        S.shard_render(b, frame[:3], frame[3:])
        frames.append(frame)
        if loss is not None:
            gc, gd = _upstream(loss, dL, dD)
            accs.append(S.shard_backward_render(b, gc, det, gd).clone())
    frame = torch.stack(frames).sum(0)
    radii_real = torch.cat([S.shard_slice(b.radii, b.plan) for b in bufs])
    grads = None
    if loss is not None:
        acc = accs[0].clone()
        for a in accs[1:]:
            acc += a   # ascending rank order, what reduce_scatter_ordered does
        per = [S.shard_backward_preprocess(b, acc[b.plan.base:b.plan.base + b.plan.slice_len].contiguous(),
                                           loss != "color") for b in bufs]
        grads = _named(per, "features_rest" in d)
    return frame[:3], frame[3:], radii_real, grads


def _sparse(world, rs, d, cap_mode, loss=None, dL=None, dD=None, det=False):
    from gaussianeditor_b200 import sparse_sharded as SS
    P = d["means3D"].shape[0]
    ranks = [SS.SparseRank(S.ShardPlan(P, world, r), torch.device("cuda"), rs.image_width, rs.image_height)
             for r in range(world)]
    SS.link_virtual(ranks)

    def order(cap):
        for rk in ranks:
            rk.matrix.zero_()
        steps = []
        for rk in ranks:
            args, rest = _rank_args(d, rk.plan)
            steps.append(SS.sparse_preprocess(rk, rs, *args, cap, raw_rest=rest))
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
        rk.frame.fill_(float("nan"))
    for st in steps:
        SS.sparse_render(st, st.rk.frame[:3], st.rk.frame[3:])
    for rk in ranks:
        SS.frame_broadcast(rk)
    frame = ranks[0].frame.clone()
    assert all(torch.equal(rk.frame, frame) for rk in ranks[1:])
    radii_real = torch.cat([rk.radii_local[:rk.plan.count] for rk in ranks])
    grads = None
    if loss is not None:
        gc, gd = _upstream(loss, dL, dD)
        accs = [SS.sparse_backward_render(st, gc, det, gd) for st in steps]
        for st, acc in zip(steps, accs):
            SS.sparse_return(st, acc)
        grads = _named([SS.sparse_backward_preprocess(st, loss != "color") for st in steps], "features_rest" in d)
    return frame[:3], frame[3:], radii_real, grads


FWD_CASES = [  # world, (W, H), M allocated, active degree, sparse capacity
    (1, (400, 300), 16, 3, "full"),
    (2, (333, 201), 16, 1, "tight"),          # active degree below the allocated one
    (3, (400, 300), 16, 3, "overflow"),       # features_rest slices of ranks 1, 2 start off a 16-byte boundary
    (3, (333, 201), 1, 0, "full"),            # degree 0: features_rest [n, 0, 3] passed as NULL
    (8, (400, 300), 4, 1, "tight"),
    (8, (64, 40), 16, 3, "overflow"),         # 3 tile rows: five ranks own none
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,size,M,deg,cap_mode", FWD_CASES)
def test_forward_raw_bit_identical_to_single_gpu(world, size, M, deg, cap_mode):
    rs, t = _case(size, deg)
    d = _raw_inputs(t, M)
    if world == 3 and M == 16:
        assert any(S.shard_slice(d["features_rest"], S.ShardPlan(60013, 3, r)).data_ptr() % 16 for r in range(3))
    color, depth, radii, _ = _single(rs, d, None, None, None, False, False)
    assert int((radii > 0).sum()) > 1000
    for mode in ("dense", "sparse"):
        c, dp, r, _ = _dense(world, rs, d) if mode == "dense" else _sparse(world, rs, d, cap_mode)
        assert torch.equal(c, color) and torch.equal(dp, depth), mode
        assert torch.equal(r, radii), mode


@pytest.mark.gpu
@pytest.mark.parametrize("world,M", [(3, 16), (2, 1)])
def test_dense_peer_store_raw_writes_the_records_of_the_plain_raw_preprocess(world, M):
    """gsr_shard_preprocess_p2p_raw with `world` local buffers as the peer geometry: every buffer receives the record
    bytes gsr_shard_preprocess_raw writes for the same slices (the padded tail included)."""
    lib = _lib.load()
    rs, t = _case((400, 300), 3 if M == 16 else 0)
    d = _raw_inputs(t, M)
    P = d["means3D"].shape[0]
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    gbytes = lib.gsr_geometry_bytes(plans[0].P_pad)
    peers = [torch.full((gbytes,), 0xAB, dtype=torch.uint8, device="cuda") for _ in range(world)]
    ptrs = (C.c_void_p * world)(*[p.data_ptr() for p in peers])
    ref = None
    for p in plans:
        args, rest = _rank_args(d, p)
        b = S.shard_preprocess(p, rs, *args, geom=ref.geom if ref else None, raw_rest=rest)
        ref = ref or b
        c = S._shard_cloud(p.count, b.inputs)
        radii = torch.zeros(p.P_pad, dtype=torch.int32, device="cuda")
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(lib.gsr_shard_preprocess_p2p_raw(C.byref(b.s), C.byref(c), p.P_pad, p.base, p.slice_len, ptrs,
                                                    world, p.rank, gbytes, radii.data_ptr(), st),
                   "gsr_shard_preprocess_p2p_raw")
        sl = slice(p.base, p.base + p.count)   # the padded tail has a culled record and no radius
        assert torch.equal(radii[sl], b.radii[sl])
    torch.cuda.synchronize()
    want = S.exchange_view(ref)
    for r in range(world):
        v = _lib.ExchangeView()
        _lib.check(lib.gsr_view_exchange(C.c_void_p(peers[r].data_ptr()), plans[0].P_pad, C.byref(v)), "view")
        off = v.records - peers[r].data_ptr()
        got = peers[r][off:off + plans[0].P_pad * 48].view(plans[0].P_pad, 48)
        # bytes of culled records other than the radius word are not part of the record's content
        rad = want.view(torch.int32)[:, 11]
        assert torch.equal(got.view(torch.int32)[:, 11], rad), r
        live = rad > 0
        assert torch.equal(got[live], want[live]), r
        assert int(live.sum()) > 1000


BWD_KINDS = [("raw", "color"), ("depth", "both"), ("depth", "depth"), ("raw_depth", "both"), ("raw_depth", "depth")]
BWD_WORLDS = [  # world, (W, H), M, degree, sparse capacity
    (2, (400, 300), 16, 3, "tight"),
    (3, (333, 201), 16, 2, "overflow"),
    (8, (64, 40), 1, 0, "full"),
]


def _kind_inputs(kind, t, M):
    return _raw_inputs(t, M) if kind.startswith("raw") else _act_inputs(t, M)


def _upstreams(size, seed):
    g = torch.Generator().manual_seed(seed)
    W, H = size
    return torch.rand(3, H, W, generator=g).cuda(), (torch.rand(1, H, W, generator=g) * 0.1).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("world,size,M,deg,cap_mode", BWD_WORLDS)
@pytest.mark.parametrize("kind,loss", BWD_KINDS)
def test_backward_matches_single_gpu(kind, loss, world, size, M, deg, cap_mode):
    rs, t = _case(size, deg)
    d = _kind_inputs(kind, t, M)
    dL, dD = _upstreams(size, world)
    _, _, _, ref = _single(rs, d, loss, dL, dD, kind != "raw", False)
    for mode in ("dense", "sparse"):
        g = (_dense(world, rs, d, loss, dL, dD) if mode == "dense" else _sparse(world, rs, d, cap_mode, loss, dL, dD))[3]
        assert g.keys() == ref.keys(), mode
        for k in ref:
            assert g[k].shape == ref[k].shape, (mode, k)
            assert rel_l2(g[k].cpu().numpy(), ref[k].cpu().numpy()) <= 2e-5, (mode, k)
    if loss != "color":   # the depth term really moves the means
        _, _, _, no_depth = _single(rs, d, "color", dL, dD, False, False)
        assert rel_l2(ref["means3D"].cpu().numpy(), no_depth["means3D"].cpu().numpy()) > 1e-3


def _bits_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k


DET_WORLDS = [(1, (400, 300), 16, 3, ("full", "tight")), (3, (333, 201), 16, 3, ("tight", "overflow")),
              (8, (64, 40), 4, 1, ("overflow", "full"))]


@pytest.mark.gpu
@pytest.mark.parametrize("world,size,M,deg,caps", DET_WORLDS)
@pytest.mark.parametrize("kind,loss", BWD_KINDS)
def test_deterministic_backward_repeatable_dense_equals_sparse(kind, loss, world, size, M, deg, caps):
    rs, t = _case(size, deg)
    d = _kind_inputs(kind, t, M)
    dL, dD = _upstreams(size, 10 + world)
    dense = _dense(world, rs, d, loss, dL, dD, det=True)[3]
    _bits_equal(dense, _dense(world, rs, d, loss, dL, dD, det=True)[3])                 # call to call
    sparse = _sparse(world, rs, d, caps[0], loss, dL, dD, det=True)[3]
    _bits_equal(sparse, _sparse(world, rs, d, caps[1], loss, dL, dD, det=True)[3])      # independent of the capacity
    for k in dense:
        assert torch.equal(dense[k], sparse[k]), k
    _, _, _, ref = _single(rs, d, loss, dL, dD, kind != "raw", True)
    assert dense.keys() == ref.keys()
    for k in ref:
        if world == 1:
            assert torch.equal(dense[k], ref[k]), k
        else:
            assert rel_l2(dense[k].cpu().numpy(), ref[k].cpu().numpy()) <= 2e-5, k


def _one_rank_sparse_pool(P, W, H):
    from gaussianeditor_b200 import sparse_sharded as SS
    rk = SS.SparseRank(S.ShardPlan(P, 1, 0), torch.device("cuda"), W, H)
    SS.link_virtual([rk])
    pool = SS.SparsePool.__new__(SS.SparsePool)
    pool.all, pool.free, pool.cap, pool.redo = [rk], [rk], rk.cap_alloc, 0
    return pool


def _module_grads(m, d, loss, dL, dD):
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in d.items()}
    m2 = torch.zeros_like(d["means3D"], requires_grad=True)
    if "features_rest" in d:
        color, radii, depth = m.forward_raw(leaves["means3D"], m2, leaves["opacity_logits"], leaves["features_dc"],
                                            leaves["features_rest"], leaves["log_scales"], leaves["raw_rotations"])
    else:
        color, radii, depth = m(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"],
                                shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"])
    _loss(loss, color, depth, dL, dD).backward()
    g = {k: v.grad for k, v in leaves.items()}
    g["means2D"] = m2.grad
    return color.detach(), depth.detach(), radii, g


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["dense", "sparse"])
@pytest.mark.parametrize("raw", [False, True])
def test_module_depth_grad_semantics_at_one_rank(mode, raw):
    """The autograd functions through the module (a one-rank group): deterministic, a colour + depth loss and a depth-only
    loss give GaussianRasterizer(depth_grad=True, deterministic=True)'s bits (a None colour gradient becomes zeros), and
    with depth_grad=True a colour-only loss gives the depth_grad=False bits."""
    rs, t = _case((333, 201), 3)
    d = _raw_inputs(t, 16) if raw else _act_inputs(t, 16)
    P = d["means3D"].shape[0]
    dL, dD = _upstreams((333, 201), 3)
    pool = _one_rank_sparse_pool(P, 333, 201) if mode == "sparse" else None
    m = _module(rs, P, deterministic=True, depth_grad=True, mode=mode, pool=pool)
    for loss in ("both", "depth"):
        c, dp, r, g = _module_grads(m, d, loss, dL, dD)
        rc, rd, rr, rg = _single(rs, d, loss, dL, dD, True, True)
        assert torch.equal(c, rc) and torch.equal(dp, rd) and torch.equal(r, rr)
        _bits_equal(g, rg)
    off = _module(rs, P, deterministic=True, depth_grad=False, mode=mode, pool=pool)
    _bits_equal(_module_grads(m, d, "color", dL, dD)[3], _module_grads(off, d, "color", dL, dD)[3])
    # depth_grad=False drops the depth gradient, as GaussianRasterizer does
    _bits_equal(_module_grads(off, d, "both", dL, dD)[3], _module_grads(off, d, "color", dL, dD)[3])


def _torchrun(variant, nproc):
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    args = {"dense-nccl": [], "dense-p2p": ["--p2p"], "sparse": ["--mode", "sparse"]}[variant]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sharded_check.py"), "--config", "c3",
           "--P", "30001", "--raw", "--depth-grad"] + args
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    child = "\n".join(l for l in r.stderr.splitlines() if l.startswith("[rank"))
    assert r.returncode == 0, r.stdout[-2000:] + child[-3000:] + r.stderr[-2000:]
    assert "SHARDED_CHECK_OK" in r.stdout and "fused_depth=ok" in r.stdout, r.stdout[-2000:]


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
@pytest.mark.parametrize("variant", ["dense-nccl", "dense-p2p", "sparse"])
def test_torchrun_sharded_check_raw_depth_grad(variant, nproc):
    """forward_raw with depth_grad=True under torchrun, one process per GPU: frames bit-identical to one GPU, gradients
    of a colour + depth loss and of a depth-only loss within tolerance."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    _torchrun(variant, nproc)
