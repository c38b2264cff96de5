"""Deterministic mode of the Gaussian-sharded rasterizer (dense and sparse exchange).

CPU: the deterministic sharded entry points are exported and bound and reject bad arguments before touching a device;
the owner form of the emission slot (common.cuh, built for the host) maps a rank's instances one-to-one onto
[0, R_rank) in the order the sharded binning emits them, on the CPU oracle's forward state; the ordered
reduce-scatter over gloo equals an explicit ascending-rank sum bit for bit.
GPU: `world` virtual ranks on one GPU drive the step functions with the ordered sum of the ranks' partial rows. For a
fixed world size the results are the same bits from call to call, do not depend on the sparse segment capacity, and
dense equals sparse; at world 1 both equal GaussianRasterizer(deterministic=True); at larger worlds the gradients are
within the sharded tolerance of it, `cnt` is bit-identical and `weights` are bit-identical with binary masks. The module
runs under torchrun and torch's deterministic flag through tools/sharded_check.py --deterministic.
"""
import ctypes as C
import os
import shutil
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gaussianeditor_b200 import _lib, sharded as S, synth
from util import cloud_tensors, rel_l2, settings_from

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, WORKSPACE = -1, -3  # GSR_ERR_INVALID, GSR_ERR_WORKSPACE
DET_NAMES = ("gsr_shard_backward_render_deterministic", "gsr_shard_apply_weights_deterministic")


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_deterministic_entry_points_are_exported_and_bound():
    lib = _lib.load()
    for name in DET_NAMES:
        assert name in _lib.SYMBOLS
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and fn.argtypes is not None


def _settings():
    d = C.c_void_p(256)
    return _lib.Settings(64, 64, 1.0, 1.0, 1.0, 0, 1, 0, 0, d, d, d, d), d


def test_shard_backward_render_deterministic_validates_before_touching_the_device():
    lib = _lib.load()
    s, d = _settings()
    P, R = 100, 10
    need = lib.gsr_deterministic_scratch_bytes(P, R, 0)
    assert need > 0

    def call(owner=_lib.TileOwner(2, 1), P=P, R=R, det=d, dbytes=need):
        return lib.gsr_shard_backward_render_deterministic(C.byref(s), C.byref(owner), P, R, d, 1 << 20, d, 1 << 20, d,
                                                           1 << 20, d, d, 1 << 20, det, dbytes, None)
    assert call(det=None) == WORKSPACE and b"deterministic scratch" in lib.gsr_last_error()
    assert call(dbytes=need - 1) == WORKSPACE and b"deterministic scratch" in lib.gsr_last_error()
    for stride, phase in [(2, 2), (0, 0), (3, -1)]:
        assert call(owner=_lib.TileOwner(stride, phase)) == INVALID and b"row_stride" in lib.gsr_last_error()
    assert call(R=-1) == INVALID and call(P=0) == INVALID


def test_shard_apply_weights_deterministic_validates_before_touching_the_device():
    lib = _lib.load()
    s, d = _settings()
    P, R = 100, 10

    def call(owner=_lib.TileOwner(2, 1), CH=1, ws=None, cs=1, P=P, R=R, det=d, dbytes=None):
        ws = CH if ws is None else ws
        dbytes = lib.gsr_deterministic_scratch_bytes(P, max(R, 0), CH) if dbytes is None else dbytes
        return lib.gsr_shard_apply_weights_deterministic(C.byref(s), C.byref(owner), P, R, d, 1 << 20, d, 1 << 20, d,
                                                         1 << 20, d, d, CH, d, ws, d, cs, det, dbytes, None)
    for CH in (1, 2, 3):
        assert call(CH=CH, ws=12) == INVALID and b"weights_stride" in lib.gsr_last_error()
    assert call(CH=0) == INVALID and call(CH=4) == INVALID
    assert call(det=None) == WORKSPACE and b"deterministic scratch" in lib.gsr_last_error()
    need = lib.gsr_deterministic_scratch_bytes(P, R, 3)
    assert call(CH=3, dbytes=need - 1) == WORKSPACE
    for stride, phase in [(2, 2), (0, 0), (3, -1)]:
        assert call(owner=_lib.TileOwner(stride, phase)) == INVALID and b"row_stride" in lib.gsr_last_error()
    assert call(R=-1) == INVALID and call(cs=0) == INVALID
    assert call(R=0) == 0   # nothing to walk: no device work, outputs untouched


_SLOT_LIB = {}


def _slot_lib(tmp_dir):
    """tests/emission_slot_host.cpp, built for the host from the kernels' header into a temporary directory."""
    if "lib" not in _SLOT_LIB:
        gxx = shutil.which("g++")
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
        if gxx is None or not os.path.exists(os.path.join(inc, "cuda_runtime.h")):
            pytest.skip("needs g++ and the CUDA headers")
        out = os.path.join(tmp_dir, "libemission_slot_host.so")
        subprocess.check_call([gxx, "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC",
                               "-I" + inc, "-o", out, os.path.join(ROOT, "tests", "emission_slot_host.cpp")])
        lib = C.CDLL(out)
        lib.owned_counts.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_int] * 4 + [C.c_void_p]
        lib.owner_slots.argtypes = [C.c_int] + [C.c_void_p] * 6 + [C.c_int] * 4 + [C.c_void_p]
        _SLOT_LIB["lib"] = lib
    return _SLOT_LIB["lib"]


def _p(a):
    return a.ctypes.data


@pytest.mark.parametrize("scene", ["c3_small", "frustum_edge", "needle"])
def test_owner_emission_slots_follow_the_sharded_emission_order(scene, tmp_path_factory):
    from oracle import cpu_oracle
    lib = _slot_lib(str(tmp_path_factory.mktemp("slot")))
    if scene == "c3_small":
        cloud, cams = synth.make_config("c3", P=3000)
        cam = cams[0]
    elif scene == "frustum_edge":
        cloud, cam = synth.frustum_edge_cloud()
    else:
        cloud, cam = synth.needle_cloud(P=300)
    f = cpu_oracle.forward_from(cloud, cam)
    try:
        P, R = f.P, f.num_rendered
        assert R > 0
        gx, gy = (f.W + 15) // 16, (f.H + 15) // 16
        px = np.ascontiguousarray(f.means2D[:, 0], np.float32)
        py = np.ascontiguousarray(f.means2D[:, 1], np.float32)
        rad = np.ascontiguousarray(f.radii, np.int32)
        depth_bits = f.depths.astype(np.float32).view(np.uint32).astype(np.uint64)
        tile_of = np.zeros(R, np.int64)
        for t, (a, b) in enumerate(f.ranges):
            tile_of[a:b] = t
        g_inst = f.point_list.astype(np.int64)
        tx_all, ty_all = tile_of % gx, tile_of // gx
        full = f.tiles_touched.astype(np.int64)
        for world in (2, 3, 8):
            covered = np.zeros(P, np.int64)
            for phase in range(world):
                touched = np.zeros(P, np.uint32)
                lib.owned_counts(P, _p(px), _p(py), _p(rad), gx, gy, world, phase, _p(touched))
                covered += touched
                mine = ty_all % world == phase   # the instances of the owned tile rows
                R_rank = int(mine.sum())
                assert int(touched.sum()) == R_rank
                # the sharded depth order: (depth bits, index) for the Gaussians with owned tiles, the others behind
                t64 = touched.astype(np.int64)
                key = np.where(t64 > 0, depth_bits, np.uint64(0xFFFFFFFF))
                order = np.lexsort((np.arange(P), key))
                excl = np.zeros(P, np.int64)
                excl[order] = np.cumsum(t64[order]) - t64[order]
                g = g_inst[mine]
                tx = np.ascontiguousarray(tx_all[mine], np.int32)
                ty = np.ascontiguousarray(ty_all[mine], np.int32)
                ex = np.ascontiguousarray(excl[g], np.uint32)
                gpx, gpy, grad = (np.ascontiguousarray(a[g]) for a in (px, py, rad))   # alive during the call
                slot = np.zeros(R_rank, np.uint32)
                lib.owner_slots(R_rank, _p(gpx), _p(gpy), _p(grad), _p(ex), _p(tx), _p(ty), gx, gy, world, phase,
                                _p(slot))
                slot = slot.astype(np.int64)
                # one-to-one onto [0, R_rank), and in emission order: Gaussians in depth order, each one's owned
                # tiles row-major (the tile id grows along a Gaussian's run)
                assert np.array_equal(np.sort(slot), np.arange(R_rank)), (world, phase)
                inv = np.empty(R_rank, np.int64)
                inv[slot] = np.arange(R_rank)
                g_by_slot = g[inv]
                tile_by_slot = (ty.astype(np.int64) * gx + tx)[inv]
                rank_of = np.empty(P, np.int64)
                rank_of[order] = np.arange(P)
                assert np.all(np.diff(rank_of[g_by_slot]) >= 0)
                same = g_by_slot[1:] == g_by_slot[:-1]
                assert np.all(np.diff(tile_by_slot)[same] > 0)
                assert np.all(slot - excl[g] < t64[g])
            # the phases together cover each Gaussian's whole rectangle
            assert np.array_equal(covered, full), world
        # {1, 0}: every tile row, the single-GPU count
        t1 = np.zeros(P, np.uint32)
        lib.owned_counts(P, _p(px), _p(py), _p(rad), gx, gy, 1, 0, _p(t1))
        assert np.array_equal(t1.astype(np.int64), full)
    finally:
        f.close()


def _gloo_ordered_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ex = S.Exchange()
        plan = S.ShardPlan(1001, world, rank)
        n = plan.slice_len
        # values of very different magnitudes: a different summation order would change the bits
        parts = []
        for r in range(world):
            g = torch.Generator().manual_seed(17 + r)
            parts.append(torch.randn(plan.P_pad, S.ACC_STRIDE, generator=g) * torch.logspace(-6, 6, S.ACC_STRIDE))
        mine = torch.empty(n, S.ACC_STRIDE)
        ex.reduce_scatter_ordered(parts[rank], mine)
        want = parts[0][rank * n:(rank + 1) * n].clone()
        for r in range(1, world):
            want += parts[r][rank * n:(rank + 1) * n]
        out[rank] = bool(torch.equal(mine.view(torch.int32), want.view(torch.int32)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_reduce_scatter_ordered_is_the_ascending_rank_sum(world):
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_gloo_ordered_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    assert [out[r] for r in range(world)] == [True] * world


# ---------------------------------------------------------------------------------------------------------------- GPU
_CLOUD = {}


def _cloud():
    if not _CLOUD:
        cloud, _ = synth.make_config("c3", P=60013)   # P not divisible by the world sizes: padded tail on the last rank
        _CLOUD["cloud"] = cloud
        _CLOUD["t"] = cloud_tensors(cloud, "cuda")
    return _CLOUD["cloud"], _CLOUD["t"]


def _cov3d(scales, rotations):
    q = rotations / rotations.norm(dim=1, keepdim=True)
    r, x, y, z = q.unbind(1)
    Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                      2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                      2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    M = Rm * scales[:, None, :]
    Sg = M @ M.transpose(1, 2)
    return torch.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], 1).contiguous()


def _inputs(t, colors, cov):
    """The per-Gaussian inputs of one case (full cloud): dict with means3D, shs, colors, opacities, scales, rotations,
    cov (empty tensors where unused)."""
    empty = torch.empty(0, device="cuda")
    P = t["means3D"].shape[0]
    d = dict(means3D=t["means3D"], opacities=t["opacities"], shs=empty, colors=empty, scales=empty, rotations=empty,
             cov=empty)
    if colors:
        g = torch.Generator().manual_seed(5)
        d["colors"] = torch.rand(P, 3, generator=g).cuda()
    else:
        d["shs"] = t["shs"]
    if cov:
        d["cov"] = _cov3d(t["scales"], t["rotations"])
    else:
        d["scales"], d["rotations"] = t["scales"], t["rotations"]
    return d


NAMES = ("means3D", "means2D", "shs", "colors", "opacities", "scales", "rotations", "cov")


def _single_grads(rs, d, dL):
    """GaussianRasterizer(deterministic=True): gradients of every used input, means2D included."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in d.items() if v.numel()}
    m2 = torch.zeros_like(d["means3D"], requires_grad=True)
    kw = dict(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], shs=leaves.get("shs"),
              colors_precomp=leaves.get("colors"), scales=leaves.get("scales"), rotations=leaves.get("rotations"),
              cov3D_precomp=leaves.get("cov"))
    color, _, _ = GaussianRasterizer(rs, deterministic=True)(**kw)
    (color * dL).sum().backward()
    out = {k: v.grad for k, v in leaves.items()}
    out["means2D"] = m2.grad
    return out


def _cat(per_rank, used):
    """per-rank gradient tuples (shard_backward_preprocess order) -> full tensors of the used inputs."""
    out = {}
    for i, name in enumerate(("means3D", "means2D", "shs", "colors", "opacities", "scales", "rotations", "cov")):
        if name in used:
            out[name] = torch.cat([g[i] for g in per_rank])
    return out


def _rank_args(d, p):
    sl = lambda k: S.shard_slice(d[k], p) if d[k].numel() else d[k]
    return (sl("means3D"), sl("shs"), sl("colors"), sl("opacities"), sl("scales"), sl("rotations"), sl("cov"))


def _aw_args(d, p):
    sl = lambda k: S.shard_slice(d[k], p) if d[k].numel() else d[k]
    empty = torch.empty(0, device="cuda")
    return (sl("means3D"), empty, sl("means3D"), sl("opacities"), sl("scales"), sl("rotations"), sl("cov"))


def _ordered_sum(parts):
    """The ranks' partial rows added in ascending rank order (what reduce_scatter_ordered does)."""
    total = parts[0].clone()
    for p in parts[1:]:
        total += p
    return total


def _dense_grads(world, rs, d, dL):
    P = d["means3D"].shape[0]
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    geom = radii = None
    bufs = []
    for p in plans:
        b = S.shard_preprocess(p, rs, *_rank_args(d, p), geom=geom, radii=radii)
        geom, radii = b.geom, b.radii
        bufs.append(b)
    for b in bufs:
        b.geom = geom.clone(); b.radii = torch.full_like(radii, -7)
    accs = []
    for b in bufs:
        S.shard_order(b)
        frame = torch.zeros(4, rs.image_height, rs.image_width, device="cuda")
        S.shard_render(b, frame[:3], frame[3:])
        accs.append(S.shard_backward_render(b, dL, deterministic=True).clone())
    acc = _ordered_sum(accs)
    grads = [S.shard_backward_preprocess(b, acc[b.plan.base:b.plan.base + b.plan.slice_len].contiguous()) for b in bufs]
    return _cat(grads, {k for k, v in d.items() if v.numel()} | {"means2D"})


def _sparse_ranks(world, W, H, P):
    from gaussianeditor_b200 import sparse_sharded as SS
    ranks = [SS.SparseRank(S.ShardPlan(P, world, r), torch.device("cuda"), W, H) for r in range(world)]
    SS.link_virtual(ranks)
    return ranks


def _sparse_order(ranks, rs, d, cap_mode, args=_rank_args):
    from gaussianeditor_b200 import sparse_sharded as SS

    def order(cap):
        for rk in ranks:
            rk.matrix.zero_()
        steps = [SS.sparse_preprocess(rk, rs, *args(d, rk.plan), cap) for rk in ranks]
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
    return steps


def _sparse_grads(world, rs, d, dL, cap_mode):
    from gaussianeditor_b200 import sparse_sharded as SS
    P = d["means3D"].shape[0]
    ranks = _sparse_ranks(world, rs.image_width, rs.image_height, P)
    steps = _sparse_order(ranks, rs, d, cap_mode)
    for st in steps:
        SS.sparse_render(st, st.rk.frame[:3], st.rk.frame[3:])
    accs = [SS.sparse_backward_render(st, dL, deterministic=True) for st in steps]
    for st, acc in zip(steps, accs):
        SS.sparse_return(st, acc)
    grads = [SS.sparse_backward_preprocess(st) for st in steps]
    return _cat(grads, {k for k, v in d.items() if v.numel()} | {"means2D"})


def _bits_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k


def _equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


BWD_CASES = [  # world, sparse capacities (first, second), colours, precomputed covariance, (W, H)
    (1, ("full", "tight"), False, False, (400, 300)),
    (1, ("tight", "overflow"), True, True, (333, 201)),
    (2, ("full", "tight"), False, False, (400, 300)),
    (3, ("tight", "overflow"), True, False, (333, 201)),
    (8, ("overflow", "full"), False, True, (400, 300)),
    (8, ("tight", "full"), False, False, (64, 40)),      # 3 tile rows: five ranks own none
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,caps,colors,cov,size", BWD_CASES)
def test_backward_repeatable_dense_equals_sparse(world, caps, colors, cov, size):
    cloud, t = _cloud()
    cam = synth.ring_cameras(8, 4.5, 15.0, size[0], size[1], 61.0)[2]
    rs = settings_from(cam, (0.2, 0.5, 0.1), cloud.sh_degree, "cuda")
    d = _inputs(t, colors, cov)
    g = torch.Generator().manual_seed(world)
    dL = torch.rand(3, size[1], size[0], generator=g).cuda()
    ref = _single_grads(rs, d, dL)
    dense = _dense_grads(world, rs, d, dL)
    _bits_equal(dense, _dense_grads(world, rs, d, dL))                  # call to call
    sparse = _sparse_grads(world, rs, d, dL, caps[0])
    _bits_equal(sparse, _sparse_grads(world, rs, d, dL, caps[1]))       # independent of the segment capacity
    _equal(dense, sparse)                                               # the same partial rows, the same order
    assert dense.keys() == ref.keys()
    if world == 1:
        _equal(dense, ref)
    else:
        for k in ref:
            assert rel_l2(dense[k].cpu().numpy(), ref[k].cpu().numpy()) <= 2e-5, k


def _mask(CH, H, W, binary, seed):
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(CH, H, W, generator=g)
    return ((m > 0.5).float() if binary else m).cuda()


def _aw_single(rs, d, iw):
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    P, CH = d["means3D"].shape[0], iw.shape[0]
    w = torch.zeros(P, CH, device="cuda"); c = torch.zeros(P, 1, dtype=torch.int32, device="cuda")
    GaussianRasterizer(rs, deterministic=True).apply_weights(
        d["means3D"], None, d["opacities"], None, w, d["scales"] if d["scales"].numel() else None,
        d["rotations"] if d["rotations"].numel() else None, d["cov"] if d["cov"].numel() else None, c, iw)
    return w, c


def _aw_dense(world, rs, d, iw):
    P, CH = d["means3D"].shape[0], iw.shape[0]
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    geom = radii = None
    bufs = []
    for p in plans:
        b = S.shard_preprocess(p, rs, *_aw_args(d, p), geom=geom, radii=radii)
        geom, radii = b.geom, b.radii
        bufs.append(b)
    for b in bufs:
        b.geom = geom.clone(); b.radii = torch.full_like(radii, -7)
    ws, cs = [], []
    for b in bufs:
        S.shard_order(b)
        wt = torch.zeros(plans[0].P_pad, CH, device="cuda")
        ct = torch.zeros(plans[0].P_pad, dtype=torch.int32, device="cuda")
        S.shard_apply_weights(b, iw, wt, ct, deterministic=True)
        ws.append(wt); cs.append(ct)
    return _ordered_sum(ws)[:P], _ordered_sum(cs)[:P, None]


def _aw_sparse(world, rs, d, iw, cap_mode):
    from gaussianeditor_b200 import sparse_sharded as SS
    P, CH = d["means3D"].shape[0], iw.shape[0]
    ranks = _sparse_ranks(world, 128, 96, P)      # apply_weights does not depend on the construction-time frame
    steps = _sparse_order(ranks, rs, d, cap_mode, _aw_args)
    accs = []
    for st in steps:
        acc = torch.zeros(world * st.cap, S.ACC_STRIDE, device="cuda")
        SS.apply_weights_walk(st, iw, acc, deterministic=True)
        accs.append(acc)
    for st, acc in zip(steps, accs):
        SS.sparse_return(st, acc)
    out_w, out_c = [], []
    for st in steps:
        w = torch.zeros(st.rk.plan.count, CH, device="cuda"); c = torch.zeros(st.rk.plan.count, 1, dtype=torch.int32,
                                                                             device="cuda")
        SS.apply_weights_gather(st, w, c)
        out_w.append(w); out_c.append(c)
    return torch.cat(out_w), torch.cat(out_c)


AW_CASES = [  # world, sparse capacity, CH, binary, cov, (W, H)
    (1, "full", 1, True, False, (400, 300)),
    (1, "tight", 3, False, False, (333, 201)),
    (2, "tight", 1, False, False, (400, 300)),
    (3, "overflow", 2, True, False, (333, 201)),
    (3, "full", 3, False, True, (400, 300)),
    (8, "tight", 2, True, True, (400, 300)),
    (8, "overflow", 3, False, False, (64, 40)),    # 3 tile rows: five ranks own none
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,cap_mode,CH,binary,cov,size", AW_CASES)
def test_apply_weights_repeatable_dense_equals_sparse(world, cap_mode, CH, binary, cov, size):
    cloud, t = _cloud()
    cam = synth.ring_cameras(8, 4.5, 15.0, size[0], size[1], 61.0)[1]
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
    d = _inputs(t, True, cov)
    iw = _mask(CH, size[1], size[0], binary, seed=world * 10 + CH)
    w_ref, c_ref = _aw_single(rs, d, iw)
    assert int((c_ref > 0).sum()) > 100
    wd, cd = _aw_dense(world, rs, d, iw)
    wd2, cd2 = _aw_dense(world, rs, d, iw)
    assert torch.equal(wd.view(torch.int32), wd2.view(torch.int32)) and torch.equal(cd, cd2)
    ws, cs = _aw_sparse(world, rs, d, iw, cap_mode)
    ws2, cs2 = _aw_sparse(world, rs, d, iw, "full" if cap_mode != "full" else "tight")
    assert torch.equal(ws.view(torch.int32), ws2.view(torch.int32)) and torch.equal(cs, cs2)
    assert torch.equal(wd, ws) and torch.equal(cd, cs)
    assert torch.equal(cd, c_ref)
    if world == 1 or binary:
        assert torch.equal(wd, w_ref)
    else:
        assert rel_l2(wd.cpu().numpy(), w_ref.cpu().numpy()) <= 1e-5


@pytest.mark.gpu
def test_config5_trace_twice_same_mask():
    """GaussianEditor's update_mask shape: 48 views at 512x512 with binary masks at world 3, twice, dense and sparse:
    identical weights, counts and thresholded masks, equal to each other and (cnt, binary weights) to one GPU."""
    cloud, cams = synth.make_config("c5", P=100_003)
    t = cloud_tensors(cloud, "cuda")
    d = _inputs(t, True, False)
    P = cloud.means3D.shape[0]
    runs = []
    for _ in range(2):
        acc = {m: [torch.zeros(P, 1, device="cuda"), torch.zeros(P, 1, dtype=torch.int32, device="cuda")]
               for m in ("dense", "sparse", "single")}
        for i, cam in enumerate(cams):
            assert (cam.image_width, cam.image_height) == (512, 512)
            rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
            yy, xx = torch.meshgrid(torch.arange(512, device="cuda"), torch.arange(512, device="cuda"), indexing="ij")
            iw = ((((xx - 256 - 3 * (i % 5)) ** 2 + (yy - 240) ** 2) < 150 ** 2).float())[None]
            for m, (w, c) in (("dense", _aw_dense(3, rs, d, iw)), ("sparse", _aw_sparse(3, rs, d, iw, "tight")),
                              ("single", _aw_single(rs, d, iw))):
                acc[m][0] += w; acc[m][1] += c
        runs.append(acc)
    for m in ("dense", "sparse"):
        for r in runs:
            assert torch.equal(r[m][0], r["single"][0]) and torch.equal(r[m][1], r["single"][1])
        assert torch.equal(runs[0][m][0].view(torch.int32), runs[1][m][0].view(torch.int32))
        assert torch.equal(runs[0][m][1], runs[1][m][1])
        masks = [(r[m][0] / (r[m][1] + 1e-7)) > 0.8 for r in runs]
        assert torch.equal(masks[0], masks[1]) and int(masks[0].sum()) > 100


def _torchrun(variant, nproc, extra=()):
    args = {"dense-nccl": [], "dense-p2p": ["--p2p"], "sparse": ["--mode", "sparse"]}[variant]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tools", "sharded_check.py"), "--config",
           "c3", "--P", "30001", "--deterministic"] + args + list(extra)
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    child = "\n".join(l for l in r.stderr.splitlines() if l.startswith("[rank"))   # the children's own traceback
    assert r.returncode == 0, r.stdout[-2000:] + child[-3000:]
    assert "SHARDED_CHECK_OK" in r.stdout and "deterministic=ok" in r.stdout
    return r.stdout.split("DETERMINISTIC_DIGEST", 1)[1].split()[0]


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
def test_torchrun_sharded_check_deterministic(nproc):
    """The module under torch's deterministic flag, one process per GPU: every variant repeats its bits (at world 1 the
    single-GPU deterministic bits), and all variants give the same digest, with fill_uninitialized_memory on and off."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    digests = {v: _torchrun(v, nproc) for v in ("dense-nccl", "dense-p2p", "sparse")}
    digests["sparse-nofill"] = _torchrun("sparse", nproc, ["--no-fill"])
    digests["dense-nofill"] = _torchrun("dense-nccl", nproc, ["--no-fill"])
    assert len(set(digests.values())) == 1, digests
