"""Fixed-capacity forward of the Gaussian-sharded rasterizer (`ShardedGaussianRasterizer(static_capacity=N)`).

CPU: the entry points (gsr_shard_order_static, gsr_sparse_order_static, gsr_shard_render_static, gsr_shard_static_gate,
gsr_peer_barrier_device) are declared, exported and bound; bad arguments are rejected before any launch; the new
control-block offsets match the Python constants and fit the block; the constructor rejects bad options before any
collective (single-process gloo group).
GPU, one device: VIRTUAL ranks (worlds 1/2/3/8, dense and sparse) at capacities of exactly max R and 1.25 R + 4096, with
and without deterministic mode, alpha and depth: frames, radii and alpha are the single-GPU bits, the ranks' R add up to
the single-GPU R and the gradients equal the default sharded path (bit for bit when deterministic). Overflow of one
rank's R, of a segment, and of both: every rank's frame is empty, every gradient exactly zero, and the status words give
every rank the right message. The device-epoch barrier on two virtual ranks and two streams: counters advance by one,
matrix rows and status words land everywhere, the error word stays 0. World 1 (and 2 with two GPUs) through torchrun:
tools/sharded_check.py --static, the eager static step equals the default one and a captured + replayed step equals
the eager calls bit for bit.
"""
import ctypes as C
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gaussianeditor_b200 import _lib, sharded as S, sparse_sharded as SS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID, WORKSPACE = -1, -3  # GSR_ERR_INVALID, GSR_ERR_WORKSPACE
D = C.c_void_p(256)          # a 16-byte aligned fake device pointer: nothing may dereference it
BIG = 1 << 30
NAMES = {"gsr_shard_order_static": 7, "gsr_sparse_order_static": 7, "gsr_shard_render_static": 18,
         "gsr_shard_static_gate": 14, "gsr_peer_barrier_device": 6}


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_entry_points_are_declared_exported_and_bound():
    header = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    lib = _lib.load()
    for name, nargs in NAMES.items():
        assert re.search(r"GSR_API int " + name + r"\(", header), name
        assert name in _lib.SYMBOLS
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == nargs, name


def test_control_block_offsets_match_and_fit():
    header = open(os.path.join(ROOT, "include", "gsr_b200.h")).read()
    defs = {k: int(v) for k, v in re.findall(r"#define (GSR_PEER_CTRL_\w+) (\d+)", header)}
    assert defs["GSR_PEER_CTRL_BYTES"] == SS.CTRL_BYTES
    assert defs["GSR_PEER_CTRL_EPOCH_OFFSET"] == SS.CTRL_EPOCH_OFFSET
    assert defs["GSR_PEER_CTRL_STATUS_OFFSET"] == SS.CTRL_STATUS_OFFSET
    matrix_end = defs["GSR_PEER_CTRL_MATRIX_OFFSET"] + 4 * SS.MAXP * SS.MAXP
    assert matrix_end <= SS.CTRL_EPOCH_OFFSET and SS.CTRL_EPOCH_OFFSET + 4 <= SS.CTRL_STATUS_OFFSET
    assert SS.CTRL_STATUS_OFFSET + 4 * SS.MAXP <= SS.CTRL_BYTES
    assert SS.CTRL_EPOCH_OFFSET % 4 == 0 and SS.CTRL_STATUS_OFFSET % 4 == 0


def _err(rc, want, text):
    assert rc == want, (rc, _lib.load().gsr_last_error())
    assert text.encode() in _lib.load().gsr_last_error(), _lib.load().gsr_last_error()


def _settings(W=64, H=48):
    return _lib.Settings(H, W, 1.0, 1.0, 1.0, 3, 16, 0, 0, D, D, D, D)


def test_static_entry_points_validate_before_any_launch():
    lib = _lib.load()
    s, own = _settings(), _lib.TileOwner(2, 1)

    def render(cap=100, status=D, counts=None, world=0, seg_cap=0, P=1000):
        return lib.gsr_shard_render_static(C.byref(s), C.byref(own), P, cap, D, BIG, D, BIG, D, BIG, D, D, D, status,
                                           counts, world, seg_cap, None)
    for cap in (0, -3):
        _err(render(cap=cap), INVALID, "static capacity must be positive")
    _err(render(status=None), INVALID, "status is null")
    _err(render(counts=D, world=2, seg_cap=501), INVALID, "world*seg_cap == P_total")    # seg_cap past the workspace
    _err(render(counts=D, world=9, seg_cap=100, P=900), INVALID, "world*seg_cap == P_total")
    _err(render(counts=D, world=2, seg_cap=0), INVALID, "world*seg_cap == P_total")
    _err(lib.gsr_shard_render_static(C.byref(s), C.byref(_lib.TileOwner(2, 2)), 1000, 100, D, BIG, D, BIG, D, BIG, D, D,
                                     D, D, None, 0, 0, None), INVALID, "tile owner")
    _err(lib.gsr_shard_order_static(C.byref(s), C.byref(own), 1000, None, BIG, D, None), INVALID, "shard_order")
    _err(lib.gsr_shard_order(C.byref(s), C.byref(own), 1000, D, BIG, D, None, None), INVALID, "shard_order")  # host word
    plan = _lib.SparsePlan(2, 0, 500, 0)
    _err(lib.gsr_sparse_order_static(C.byref(s), C.byref(plan), D, BIG, D, D, None), INVALID, "sparse plan")
    plan = _lib.SparsePlan(2, 0, 500, 100)
    _err(lib.gsr_sparse_order_static(C.byref(s), C.byref(plan), D, BIG, None, D, None), INVALID, "null argument")
    _err(lib.gsr_sparse_order(C.byref(s), C.byref(plan), D, BIG, D, D, None, None), INVALID, "null argument")

    def gate(flags=D, n=2, flag_sum=None, planes=4, status=D, ibytes=BIG):
        return lib.gsr_shard_static_gate(C.byref(s), 1000, D, BIG, D, ibytes, flags, n, flag_sum, None, D, planes,
                                         status, None)
    _err(gate(status=None), INVALID, "bad arguments")
    _err(gate(flags=None), INVALID, "exactly one of flags")
    _err(gate(flag_sum=D), INVALID, "exactly one of flags")
    _err(gate(n=9), INVALID, "exactly one of flags")
    _err(gate(planes=3), INVALID, "planes")
    _err(gate(ibytes=64), WORKSPACE, "image workspace too small")
    arr = (C.c_void_p * 2)(D, None)
    _err(lib.gsr_peer_barrier_device(2, 0, arr, 0, None, None), INVALID, "peer block 1 is null")
    _err(lib.gsr_peer_barrier_device(2, 2, arr, 0, None, None), INVALID, "bad arguments")


def test_status_messages_name_what_overflowed():
    assert S.static_status_error([10, 0, 0, 0], 100, None, 0) is None
    assert "R=150 exceeds static_capacity=100" in S.static_status_error([150, 1, 0, 0], 100, None, 1)
    assert "another rank" in S.static_status_error([50, 1, 0, 0], 100, None, 1)
    assert "another rank" in S.static_status_error([50, 1, 30, 0], 100, 40, 1)
    assert "segment of 50 records exceeds segment_capacity=40" in S.static_status_error([50, 1, 50, 0], 100, 40, 0)
    assert "timed out" in S.static_status_error([50, 0, 0, 1], 100, 40, 0)


def _ctor_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from gaussianeditor_b200 import gaussian_renderer as GR
        z = torch.zeros

        def rs(debug=False):
            return GR.GaussianRasterizationSettings(48, 64, 1.0, 1.0, z(3), 1.0, torch.eye(4), torch.eye(4), 0, z(3),
                                                    False, debug)
        ok = True

        def raises(match, **kw):
            try:
                S.ShardedGaussianRasterizer(kw.pop("settings", rs()), 100, **kw)
            except ValueError as e:
                return match in str(e)
            return False
        for bad in (0, -1, 2.5, True, 2 ** 31, "7", [3]):
            ok &= raises("static_capacity", mode="dense", p2p=False, static_capacity=bad)
        for bad in (0, 2.5, False, 2 ** 31):
            ok &= raises("segment_capacity", mode="sparse", static_capacity=10, segment_capacity=bad)
        ok &= raises("segment_capacity", mode="sparse", static_capacity=10, segment_capacity=101)   # > the allocation
        ok &= raises("mode='sparse' only", mode="dense", p2p=False, static_capacity=10, segment_capacity=5)
        ok &= raises("needs static_capacity", mode="sparse", segment_capacity=5)
        ok &= raises("debug", settings=rs(True), mode="dense", p2p=False, static_capacity=10)
        ok &= S.check_static_options(1000.0, None, None, rs()) == (1000, None)
        ok &= S.check_static_options(None, None, "dense", rs(True)) == (None, None)
        out[rank] = ok
    finally:
        dist.destroy_process_group()


def test_constructor_validates_before_any_collective():
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_ctor_worker, args=(1, _free_port(), out), nprocs=1, join=True)
    assert out[0] is True


# ---------------------------------------------------------------------------------------------------------------- GPU
def _setup(world):
    from test_sharded import _case
    from util import cloud_tensors, settings_from
    case = _case()
    dev = torch.device("cuda")
    cloud, cam, bg = case["cloud"], case["cam"], case["bg"]
    H, W = cam.image_height, cam.image_width
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    full = cloud_tensors(cloud, dev)
    g = np.random.default_rng(5)
    up = dict(color=torch.from_numpy(case["dL"]).to(dev),
              depth=torch.from_numpy(g.random((1, H, W), dtype=np.float32) * 0.1).to(dev),
              alpha=torch.from_numpy(g.random((1, H, W), dtype=np.float32) - 0.5).to(dev))
    return case, rs, full, up, [S.ShardPlan(cloud.means3D.shape[0], world, r) for r in range(world)]


NAMES8 = ["dmean3D", "dmean2D", "dsh", None, "dopacity", "dscale", "drot", None]


def _dense(case, rs, full, up, plans, capacity, det, depth):
    """One dense step on virtual ranks; capacity None = the default path. Returns (frames [world] of [5,H,W], radii,
    statuses, per-rank gradient tuples)."""
    dev = torch.device("cuda")
    P = full["means3D"].shape[0]
    H, W = int(rs.image_height), int(rs.image_width)
    empty = torch.empty(0, device=dev)
    geom = radii = None
    bufs = []
    for p in plans:
        sl = lambda t: S.shard_slice(t, p)
        b = S.shard_preprocess(p, rs, sl(full["means3D"]), sl(full["shs"]), empty, sl(full["opacities"]),
                               sl(full["scales"]), sl(full["rotations"]), empty, geom=geom, radii=radii)
        geom, radii = b.geom, b.radii
        bufs.append(b)
    frames, statuses = [], []
    for b in bufs:
        b.geom = geom.clone(); b.radii = torch.full_like(radii, -7)
        frame = torch.zeros(5, H, W, device=dev)
        if capacity is None:
            S.shard_order(b)
            S.shard_render(b, frame[:3], frame[3:4])
        else:
            st = torch.full((4,), -1, dtype=torch.int32, device=dev)
            S.shard_order_static(b, capacity)
            S.shard_render_static(b, frame[:3], frame[3:4], st)
            statuses.append(st)
        S.shard_alpha(b, frame[4:])
        frames.append(frame)
    total = torch.stack(frames).sum(0)             # the all-reduce
    outs = [total.clone() for _ in bufs]
    if capacity is not None:
        flag_sum = torch.stack([st[1] for st in statuses]).sum().float().view(1)   # the flag word of the all-reduce
        for b, st, o in zip(bufs, statuses, outs):
            S.static_gate(b.s, b.plan.P_pad, b.geom, b.img, o, st, flag_sum=flag_sum)
    accs = [S.shard_backward_render(b, up["color"], det, up["depth"] if depth else None, up["alpha"]) for b in bufs]
    acc = accs[0].clone()
    for a in accs[1:]:
        acc += a                                     # ascending rank order, as reduce_scatter_ordered
    grads = [S.shard_backward_preprocess(b, acc[b.plan.base:b.plan.base + b.plan.slice_len].contiguous(), depth)
             for b in bufs]
    torch.cuda.synchronize()
    return outs, [b.radii[:P] for b in bufs], statuses, grads


def _sparse(case, rs, full, up, plans, capacity, det, depth, seg_cap=None):
    """One sparse step on virtual ranks (matrix summed and status words copied on the host, as the barriers would);
    capacity None = the default path. Returns (frames, radii_local, statuses, gradient tuples, largest segment)."""
    dev = torch.device("cuda")
    H, W = int(rs.image_height), int(rs.image_width)
    empty = torch.empty(0, device=dev)
    ranks = [SS.SparseRank(p, dev, W, H, alpha=True) for p in plans]
    SS.link_virtual(ranks)
    cap = seg_cap if seg_cap is not None else ranks[0].cap_alloc
    for rk in ranks:
        rk.matrix.zero_()
    steps = []
    for rk in ranks:
        sl = lambda t: S.shard_slice(t, rk.plan)
        steps.append(SS.sparse_preprocess(rk, rs, sl(full["means3D"]), sl(full["shs"]), empty, sl(full["opacities"]),
                                          sl(full["scales"]), sl(full["rotations"]), empty, cap))
    matrix = torch.stack([rk.matrix for rk in ranks]).sum(0)
    for rk in ranks:
        rk.matrix.copy_(matrix)
    statuses = []
    for st in steps:
        if capacity is None:
            SS.sparse_order(st)
            SS.sparse_render(st, st.rk.frame[:3], st.rk.frame[3:4])
        else:
            status = torch.full((4,), -1, dtype=torch.int32, device=dev)
            st.rk = S.StaticScratch(st.rk)
            SS.sparse_order_static(st, capacity)
            SS.sparse_render_static(st, st.rk.frame[:3], st.rk.frame[3:4], status)
            statuses.append(status)
        SS.sparse_alpha(st, st.rk.frame[4:5])
    for rk in ranks:
        SS.frame_broadcast(rk)
    outs = [rk.frame.clone() for rk in ranks]
    if capacity is not None:
        flags = torch.stack([s[1] for s in statuses])
        for rk in ranks:
            rk.status_array.copy_(flags)              # what the frame barrier's status words deliver
        for st, status, o in zip(steps, statuses, outs):
            SS.sparse_static_gate(st, o, status)
    accs = [SS.sparse_backward_render(st, up["color"], det, up["depth"] if depth else None, up["alpha"]) for st in steps]
    for st, acc in zip(steps, accs):
        SS.sparse_return(st, acc)
    grads = [SS.sparse_backward_preprocess(st, depth) for st in steps]
    torch.cuda.synchronize()
    radii = [rk.radii_local[:rk.plan.count].clone() for rk in ranks]
    return outs, radii, statuses, grads, int(matrix.max())


def _grads_match(got, want, det, tag):
    from util import rel_l2
    for gs, ws in zip(got, want):
        for name, g, w in zip(NAMES8, gs, ws):
            if name is None:
                continue
            if det:
                assert torch.equal(g, w), (tag, name)
            else:
                assert rel_l2(g.cpu().numpy(), w.cpu().numpy()) <= 2e-5, (tag, name)


def _alpha_ref(case, rs, full):
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    return GaussianRasterizer(rs, return_alpha=True)(
        means3D=full["means3D"], means2D=torch.zeros_like(full["means3D"]), opacities=full["opacities"],
        shs=full["shs"], scales=full["scales"], rotations=full["rotations"])[3]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("mode", ["dense", "sparse"])
def test_virtual_ranks_static_equals_single_gpu_and_default(world, mode):
    case, rs, full, up, plans = _setup(world)
    ref = case["ref"]
    alpha_ref = _alpha_ref(case, rs, full)
    run = _dense if mode == "dense" else _sparse
    for det in (False, True):
        for depth in (False, True):
            base = run(case, rs, full, up, plans, None, det, depth)
            Rs = None
            for which in ("exact", "headroom"):
                if Rs is None:   # per-rank R from a static run with an ample capacity
                    probe = run(case, rs, full, up, plans, 4 * ref["R"] + 4096, det, depth)
                    Rs = [int(s[0]) for s in probe[2]]
                cap = max(Rs) if which == "exact" else int(1.25 * max(Rs)) + 4096
                out = run(case, rs, full, up, plans, cap, det, depth)
                tag = (mode, world, det, depth, which)
                assert sum(int(s[0]) for s in out[2]) == ref["R"], tag
                assert all(int(s[1]) == 0 and int(s[3]) == 0 for s in out[2]), tag
                for f in out[0]:
                    assert torch.equal(f[:3], ref["color"]) and torch.equal(f[3:4], ref["depth"]), tag
                    assert torch.equal(f[4:5], alpha_ref), tag
                if mode == "dense":
                    assert all(torch.equal(r, ref["radii"]) for r in out[1]), tag
                else:
                    assert torch.equal(torch.cat(out[1]), ref["radii"]), tag
                    assert all(int(s[2]) == base[4] for s in out[2]), tag
                _grads_match(out[3], base[3], det, tag)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["R", "segment", "both"])
def test_virtual_ranks_overflow_empties_every_frame_and_zeroes_every_gradient(what):
    world = 3
    case, rs, full, up, plans = _setup(world)
    ref = case["ref"]
    probe = _sparse(case, rs, full, up, plans, 4 * ref["R"] + 4096, True, False)
    Rs, maxc = [int(s[0]) for s in probe[2]], probe[4]
    # "R": only the rank with the largest R overflows (the others fit), so they learn it from the gate alone
    assert sorted(Rs)[-1] > sorted(Rs)[-2]
    cap = {"R": max(Rs) - 1, "segment": 4 * ref["R"] + 4096, "both": 64}[what]
    seg = {"R": None, "segment": maxc // 2, "both": maxc // 2}[what]
    bg = torch.tensor(case["bg"], dtype=torch.float32, device="cuda").view(3, 1, 1).expand(3, *ref["depth"].shape[1:])
    runs = [("sparse", _sparse(case, rs, full, up, plans, cap, det, depth, seg)) for det in (False, True)
            for depth in (False, True)]
    if what == "R":
        runs += [("dense", _dense(case, rs, full, up, plans, cap, det, True)) for det in (False, True)]
    for mode, out in runs:
        frames, _, statuses, grads = out[:4]
        for f in frames:
            assert torch.equal(f[:3], bg) and int(torch.count_nonzero(f[3:])) == 0, (mode, what)
        for gs in grads:
            for g in gs:
                assert int(torch.count_nonzero(g)) == 0, (mode, what)
        assert all(int(s[1]) == 1 for s in statuses), (mode, what)
        for r, s in enumerate(statuses):
            msg = S.static_status_error(s.cpu(), cap, seg if mode == "sparse" else None, r)
            if int(s[0]) > cap:
                assert "exceeds static_capacity" in msg and "this rank" in msg
            elif what != "R" and mode == "sparse":
                assert "segment_capacity" in msg
            else:
                assert "another rank" in msg
        if what == "R":
            assert any(int(s[0]) > cap for s in statuses) and any(int(s[0]) <= cap for s in statuses)
        if what == "both":
            assert any(int(s[0]) > cap for s in statuses)


@pytest.mark.gpu
def test_device_epoch_barrier_advances_and_delivers_rows_and_status_words():
    dev = torch.device("cuda")
    plans = [S.ShardPlan(64, 2, r) for r in range(2)]
    ranks = [SS.SparseRank(p, dev, 64, 48) for p in plans]
    SS.link_virtual(ranks)
    for rk in ranks:
        rk.device_epoch = True
    side = torch.cuda.Stream()
    words = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(2)]
    for k in range(1, 7):
        with_row, with_status = k % 2 == 1, k % 3 != 0
        for r, rk in enumerate(ranks):
            rk.matrix[r, :2] = torch.tensor([10 * k + r, 100 * k + r], dtype=torch.int32, device=dev)
            words[r].fill_(1000 * k + r)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):            # the two barrier kernels must be able to run concurrently
            SS.peer_barrier(ranks[1], with_row=with_row, status_word=words[1] if with_status else None)
        SS.peer_barrier(ranks[0], with_row=with_row, status_word=words[0] if with_status else None)
        torch.cuda.synchronize()
        for rk in ranks:
            assert int(rk.err_word[0]) == 0 and int(rk.epoch_word[0]) == k
            if with_row:
                assert rk.matrix[:2, :2].cpu().tolist() == [[10 * k, 100 * k], [10 * k + 1, 100 * k + 1]]
            if with_status:
                assert rk.status_array.cpu().tolist() == [1000 * k, 1000 * k + 1]
    with pytest.raises(RuntimeError, match="device-epoch"):
        SS.peer_barrier(SS.SparseRank(plans[0], dev, 64, 48), status_word=words[0])


def _torchrun(nproc, extra):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tools", "sharded_check.py"), "--config",
           "c3", "--P", "30001", "--static"] + extra
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "SHARDED_CHECK_OK" in r.stdout, r.stdout[-2000:]


VARIANTS = {"sparse": ["--mode", "sparse"], "dense-nccl": [], "dense-p2p": ["--p2p"]}


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_world1_static_step_equals_default_and_replays_bit_for_bit(variant):
    _torchrun(1, VARIANTS[variant])


@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_world2_static_step_equals_default_and_replays_bit_for_bit(variant):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _torchrun(2, VARIANTS[variant])
