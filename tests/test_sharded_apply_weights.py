"""Semantic tracing (apply_weights) and markVisible on the Gaussian-sharded rasterizer, dense and sparse exchange.

CPU: the new C-ABI entry points are exported and bound and reject bad arguments before touching a device; the sharded
rasterizer refuses torch's deterministic flag for apply_weights as it does for forward.
GPU: `world` virtual ranks on one GPU drive the step functions (the reduce-scatter is an explicit sum, the peer stores of
the sparse exchange go to other buffers of the same device) and must reproduce the single-GPU
``GaussianRasterizer.apply_weights``: ``cnt`` bit for bit, ``weights`` bit for bit with binary masks (the sums are
integers) and to summation order with float masks. The module itself runs under torchrun (tools/sharded_check.py).
"""
import ctypes as C
import os
import socket
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import _lib, sharded as S, synth
from util import cloud_tensors, rel_l2, settings_from

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID = -1  # GSR_ERR_INVALID


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_new_entry_points_are_exported_and_bound():
    lib = _lib.load()
    for name in ("gsr_shard_apply_weights", "gsr_sparse_apply_weights_gather"):
        assert name in _lib.SYMBOLS
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and fn.argtypes is not None


def test_shard_apply_weights_validates_before_touching_the_device():
    lib = _lib.load()
    d = C.c_void_p(256)
    s = _lib.Settings(64, 64, 1.0, 1.0, 1.0, 0, 1, 0, 0, d, d, d, d)
    own = _lib.TileOwner(2, 1)

    def call(owner=own, CH=1, w=d, ws=1, c=d, cs=1, iw=d, radii=d, P=100, R=10):
        return lib.gsr_shard_apply_weights(C.byref(s), C.byref(owner), P, R, d, 1 << 20, d, 1 << 20, d, 1 << 20, radii,
                                           iw, CH, w, ws, c, cs, None)
    for CH in (0, 4, -1):
        assert call(CH=CH, ws=4) == INVALID and b"num_channels" in lib.gsr_last_error()
    assert call(w=None) == INVALID
    assert call(c=None) == INVALID
    assert call(iw=None) == INVALID
    assert call(radii=None) == INVALID
    assert call(CH=3, ws=2) == INVALID and b"stride" in lib.gsr_last_error()
    assert call(cs=0) == INVALID and b"stride" in lib.gsr_last_error()
    assert call(P=0) == INVALID and call(R=-1) == INVALID
    for stride, phase in [(2, 2), (0, 0), (3, -1)]:
        assert call(owner=_lib.TileOwner(stride, phase)) == INVALID and b"row_stride" in lib.gsr_last_error()
    assert call(R=0) == 0   # nothing to walk: no device work, outputs untouched


def test_sparse_apply_weights_gather_validates_before_touching_the_device():
    lib = _lib.load()
    d = C.c_void_p(256)
    plan = _lib.SparsePlan(3, 1, 100, 64)

    def call(p=plan, CH=1, n=50, w=d, c=d, local=d, cand=d):
        return lib.gsr_sparse_apply_weights_gather(C.byref(p), local, 1 << 30, cand, 1 << 30, n, CH, w, c, None)
    for CH in (0, 4):
        assert call(CH=CH) == INVALID and b"num_channels" in lib.gsr_last_error()
    assert call(w=None) == INVALID and call(c=None) == INVALID
    assert call(local=None) == INVALID and call(cand=None) == INVALID
    assert call(n=101) == INVALID and call(n=-1) == INVALID
    assert call(p=_lib.SparsePlan(3, 3, 100, 64)) == INVALID       # rank >= world
    assert call(p=_lib.SparsePlan(9, 0, 100, 64)) == INVALID       # more than GSR_MAX_PEERS
    assert call(n=0) == 0   # nothing to gather


def _run_py(code):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_sharded_apply_weights_refuses_torch_deterministic_flag():
    out = _run_py("""
        import warnings, torch
        from gaussianeditor_b200 import sharded
        torch.use_deterministic_algorithms(True)
        try:
            sharded.ShardedGaussianRasterizer.apply_weights(None, None, None, None)
        except RuntimeError as e:
            assert "deterministic" in str(e) and "apply_weights" in str(e), e
            print("raised")
        torch.use_deterministic_algorithms(True, warn_only=True)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            try:   # warns, then goes on (and fails on the missing module and arguments)
                sharded.ShardedGaussianRasterizer.apply_weights(None, None, None, None)
            except (AssertionError, AttributeError):
                pass
        assert any("deterministic" in str(x.message) for x in w)
        print("warned")
    """)
    assert "raised" in out and "warned" in out


# ---------------------------------------------------------------------------------------------------------------- GPU
_CLOUD = {}


def _cloud():
    if not _CLOUD:
        cloud, _ = synth.make_config("c3", P=60013)   # P not divisible by the world sizes: padded tail on the last rank
        _CLOUD["cloud"] = cloud
        _CLOUD["t"] = cloud_tensors(cloud, "cuda")
    return _CLOUD["cloud"], _CLOUD["t"]


def _cov3d(scales, rotations):
    """[P,6] upper triangle of R S S^T R^T (the precomputed-covariance input)."""
    q = rotations / rotations.norm(dim=1, keepdim=True)
    r, x, y, z = q.unbind(1)
    Rm = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                      2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                      2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    M = Rm * scales[:, None, :]
    Sg = M @ M.transpose(1, 2)
    return torch.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], 1).contiguous()


def _mask(CH, H, W, binary, seed):
    g = torch.Generator().manual_seed(seed)
    m = torch.rand(CH, H, W, generator=g)
    return ((m > 0.5).float() if binary else m).cuda()


def _geometry(t, cov):
    if cov:
        return dict(scales=None, rotations=None, cov3Ds_precomp=_cov3d(t["scales"], t["rotations"]))
    return dict(scales=t["scales"], rotations=t["rotations"], cov3Ds_precomp=None)


def _single(rs, t, geo, iw, calls=1):
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    P, CH = t["means3D"].shape[0], iw.shape[0]
    w = torch.zeros(P, CH, device="cuda")
    c = torch.zeros(P, 1, dtype=torch.int32, device="cuda")
    for _ in range(calls):
        GaussianRasterizer(rs).apply_weights(t["means3D"], None, t["opacities"], None, w, geo["scales"], geo["rotations"],
                                             geo["cov3Ds_precomp"], c, iw)
    return w, c


def _args(t, geo, p):
    empty = torch.empty(0, device="cuda")
    sl = lambda x: S.shard_slice(x, p) if x is not None else empty
    # means3D stands in the colors_precomp slot, as in ShardedGaussianRasterizer.apply_weights
    return (sl(t["means3D"]), empty, sl(t["means3D"]), sl(t["opacities"]), sl(geo["scales"]), sl(geo["rotations"]),
            sl(geo["cov3Ds_precomp"]))


W0, C0 = 7.0, 5   # initial values of every rank's rows: rows no splat of the view hits must keep them exactly


def _dense_virtual(world, rs, t, geo, iw, calls=1):
    """Virtual ranks through the dense step functions; returns per-rank (weights, cnt) rows, started at W0 / C0."""
    P, CH = t["means3D"].shape[0], iw.shape[0]
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    out = [(torch.full((p.count, CH), W0, device="cuda"), torch.full((p.count, 1), C0, dtype=torch.int32, device="cuda"))
           for p in plans]
    for _ in range(calls):
        geom = radii = None
        bufs = []
        for p in plans:
            b = S.shard_preprocess(p, rs, *_args(t, geo, p), geom=geom, radii=radii)
            geom, radii = b.geom, b.radii
            bufs.append(b)
        for b in bufs:   # each rank continues on its own copy, as after a real all-gather
            b.geom = geom.clone(); b.radii = torch.full_like(radii, -7)
        P_pad = plans[0].P_pad
        w_sum = torch.zeros(P_pad, CH, device="cuda")
        c_sum = torch.zeros(P_pad, dtype=torch.int32, device="cuda")
        for b in bufs:
            S.shard_order(b)
            wt = torch.zeros(P_pad, CH, device="cuda")
            ct = torch.zeros(P_pad, dtype=torch.int32, device="cuda")
            S.shard_apply_weights(b, iw, wt, ct)
            w_sum += wt          # the reduce-scatter
            c_sum += ct
        assert float(w_sum[P:].abs().sum()) == 0.0 and int(c_sum[P:].abs().sum()) == 0   # padded slots never hit
        for p, (w, c) in zip(plans, out):
            w += w_sum[p.base:p.base + p.count]
            c += c_sum[p.base:p.base + p.count, None]
    return plans, out


def _sparse_virtual(world, rs, t, geo, iw, cap_mode="full", calls=1, frame=(128, 96)):
    """Virtual ranks through the sparse step functions. The ranks are built for a `frame` different from the view's
    size: apply_weights must not depend on it."""
    from gaussianeditor_b200 import sparse_sharded as SS
    P, CH = t["means3D"].shape[0], iw.shape[0]
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    ranks = [SS.SparseRank(p, torch.device("cuda"), *frame) for p in plans]
    SS.link_virtual(ranks)
    out = [(torch.full((p.count, CH), W0, device="cuda"), torch.full((p.count, 1), C0, dtype=torch.int32, device="cuda"))
           for p in plans]

    def order(cap):
        for rk in ranks:
            rk.matrix.zero_()
        steps = [SS.sparse_preprocess(rk, rs, *_args(t, geo, rk.plan), cap) for rk in ranks]
        m = torch.stack([rk.matrix for rk in ranks]).sum(0)     # the count all-gather
        for rk in ranks:
            rk.matrix.copy_(m)
        return steps, [SS.sparse_order(st) for st in steps]

    for _ in range(calls):
        cap0 = ranks[0].cap_alloc
        steps, res = order(cap0)
        maxc = res[0][1]
        if cap_mode == "tight":
            steps, res = order(max(maxc, 1))
        elif cap_mode == "overflow" and maxc > 1:
            steps, res = order(max(1, maxc // 2))
            assert all(r[1] > st.cap for r, st in zip(res, steps))     # detected on every rank alike
            steps, res = order(SS.next_capacity(maxc, cap0))
        assert all(r[1] <= st.cap for r, st in zip(res, steps))
        accs = []
        for st in steps:
            M = world * st.cap
            acc = torch.zeros(M, S.ACC_STRIDE, device="cuda")
            SS.apply_weights_walk(st, iw, acc)
            accs.append(acc)
        for st, acc in zip(steps, accs):
            SS.sparse_return(st, acc)
        for st, (w, c) in zip(steps, out):
            SS.apply_weights_gather(st, w, c)
    return plans, out


def _compare(plans, out, w_ref, c_ref, binary, calls=1):
    for p, (w, c) in zip(plans, out):
        wr = S.shard_slice(w_ref, p)
        cr = S.shard_slice(c_ref, p)
        assert torch.equal(c - C0, cr), p.rank
        untouched = (cr == 0).view(-1)
        assert bool((w[untouched] == W0).all()) and bool((c[untouched] == C0).all())
        dw = w - W0
        if binary:
            assert torch.equal(dw, wr), p.rank
        else:
            assert rel_l2(dw.cpu().numpy(), wr.cpu().numpy()) <= 1e-5, p.rank
            assert float((dw - wr).abs().max()) <= 1e-4 * max(float(wr.abs().max()), 1e-30), p.rank


DENSE_CASES = [  # world, CH, binary, cov, (W, H), calls
    (2, 1, True, False, (400, 300), 2),
    (3, 2, False, False, (400, 300), 1),
    (8, 3, True, True, (400, 300), 1),
    (3, 3, False, False, (333, 201), 2),
    (8, 1, True, False, (64, 40), 1),      # 3 tile rows: five ranks own none
]
SPARSE_CASES = [  # world, capacity, CH, binary, cov, (W, H), calls
    (2, "full", 1, True, False, (400, 300), 2),
    (3, "tight", 2, False, False, (400, 300), 1),
    (3, "overflow", 3, True, False, (333, 201), 1),
    (8, "full", 2, True, False, (333, 201), 1),
    (8, "tight", 1, False, True, (400, 300), 1),
    (8, "overflow", 3, False, False, (400, 300), 2),
    (8, "tight", 3, True, False, (64, 40), 1),   # 3 tile rows: five ranks own none
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,CH,binary,cov,size,calls", DENSE_CASES)
def test_dense_virtual_ranks_match_single_gpu(world, CH, binary, cov, size, calls):
    cloud, t = _cloud()
    cam = synth.ring_cameras(8, 4.5, 15.0, size[0], size[1], 61.0)[1]
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
    geo = _geometry(t, cov)
    iw = _mask(CH, size[1], size[0], binary, seed=world * 10 + CH)
    w_ref, c_ref = _single(rs, t, geo, iw, calls)
    assert int((c_ref > 0).sum()) > 100
    plans, out = _dense_virtual(world, rs, t, geo, iw, calls)
    _compare(plans, out, w_ref, c_ref, binary)


@pytest.mark.gpu
@pytest.mark.parametrize("world,cap_mode,CH,binary,cov,size,calls", SPARSE_CASES)
def test_sparse_virtual_ranks_match_single_gpu(world, cap_mode, CH, binary, cov, size, calls):
    cloud, t = _cloud()
    cam = synth.ring_cameras(8, 4.5, 15.0, size[0], size[1], 61.0)[1]
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
    geo = _geometry(t, cov)
    iw = _mask(CH, size[1], size[0], binary, seed=world * 10 + CH + 1)
    w_ref, c_ref = _single(rs, t, geo, iw, calls)
    assert int((c_ref > 0).sum()) > 100
    plans, out = _sparse_virtual(world, rs, t, geo, iw, cap_mode, calls)
    _compare(plans, out, w_ref, c_ref, binary)


@pytest.mark.gpu
def test_config5_trace_mask_equals_single_gpu():
    """GaussianEditor's update_mask shape: 48 views at 512x512 with binary masks, world 3, then the threshold
    weights / (cnt + 1e-7) > 0.8 on every rank's rows: the mask must equal the single-GPU one exactly."""
    cloud, cams = synth.make_config("c5", P=100_003)
    t = cloud_tensors(cloud, "cuda")
    geo = _geometry(t, False)
    P = cloud.means3D.shape[0]
    w_ref = torch.zeros(P, 1, device="cuda"); c_ref = torch.zeros(P, 1, dtype=torch.int32, device="cuda")
    dense = sparse = None
    for i, cam in enumerate(cams):
        assert (cam.image_width, cam.image_height) == (512, 512)
        rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
        yy, xx = torch.meshgrid(torch.arange(512, device="cuda"), torch.arange(512, device="cuda"), indexing="ij")
        iw = ((((xx - 256 - 3 * (i % 5)) ** 2 + (yy - 240) ** 2) < 150 ** 2).float())[None]
        from gaussianeditor_b200.rasterizer import GaussianRasterizer
        GaussianRasterizer(rs).apply_weights(t["means3D"], None, t["opacities"], None, w_ref, geo["scales"],
                                             geo["rotations"], None, c_ref, iw)
        plans, d = _dense_virtual(3, rs, t, geo, iw)
        _, s = _sparse_virtual(3, rs, t, geo, iw, "tight")
        if dense is None:
            dense = [(torch.zeros_like(w), torch.zeros_like(c)) for w, c in d]
            sparse = [(torch.zeros_like(w), torch.zeros_like(c)) for w, c in s]
        for acc, res in ((dense, d), (sparse, s)):
            for (wa, ca), (w, c) in zip(acc, res):
                wa += w - W0; ca += c - C0
    mask_ref = (w_ref / (c_ref + 1e-7)) > 0.8
    assert int(mask_ref.sum()) > 100
    for acc in (dense, sparse):
        mask = torch.cat([w / (c + 1e-7) for w, c in acc]) > 0.8
        assert torch.equal(mask, mask_ref)
        assert torch.equal(torch.cat([c for _, c in acc]), c_ref)


@pytest.mark.gpu
def test_mark_visible_per_rank_is_the_single_gpu_slice():
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    cloud, t = _cloud()
    cam = synth.ring_cameras(8, 4.5, 15.0, 400, 300, 61.0)[3]
    rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, "cuda")
    ref = GaussianRasterizer(rs).markVisible(t["means3D"])
    assert 0 < int(ref.sum()) < ref.numel()
    for world in (2, 3, 8):
        for r in range(world):
            p = S.ShardPlan(ref.numel(), world, r)
            assert torch.equal(S.mark_visible(rs, S.shard_slice(t["means3D"], p)), S.shard_slice(ref, p))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
@pytest.mark.parametrize("nproc", [1, 2])
@pytest.mark.parametrize("variant", ["dense-nccl", "dense-p2p", "sparse"])
def test_torchrun_sharded_check_apply_weights(variant, nproc):
    """ShardedGaussianRasterizer.apply_weights / markVisible through the module, one process per GPU (world 1 runs
    every collective and peer mapping of the path on a single GPU)."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    extra = {"dense-nccl": [], "dense-p2p": ["--p2p"], "sparse": ["--mode", "sparse"]}[variant]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tools", "sharded_check.py"), "--config",
           "c3", "--P", "30001", "--apply-weights"] + extra
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "SHARDED_CHECK_OK" in r.stdout and "apply_weights" in r.stdout
