"""`grad_mask` on the Gaussian-sharded rasterizer: the edit bit travels in the splat record (q1.w), and the tile owners'
blend backward skips the unedited splats.

CPU: the new entry points are declared, exported and bound; each rejects a NULL mask (and a camera) before touching a
device; the module's forward checks the mask before any collective.
GPU, virtual ranks on one GPU (the step functions, dense and sparse): forward outputs are the unmasked bits, unedited
rows are +0.0, edited rows are the unmasked deterministic rows, dense equals sparse, and at world 1 the rows equal
``GaussianRasterizer(deterministic=True, grad_mask=...)``; first[] of every owned tile equals a numpy restatement.
GPU, world 1 through an NCCL group in this process: dense NCCL, dense p2p and sparse agree with the virtual ranks, a
captured static step replays bit for bit, overflow gives zeros, and ``run_sharded_edit_loop(grad_mask="kernel")`` equals
``grad_mask="hooks"``.
"""
import ctypes as C
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist

from gaussianeditor_b200 import _lib, sharded as S, synth
from util import cloud_tensors, rel_l2, settings_from

INVALID = -1  # GSR_ERR_INVALID

MASKED_ENTRY_POINTS = ("gsr_shard_preprocess_masked", "gsr_shard_preprocess_raw_masked",
                       "gsr_shard_preprocess_p2p_masked", "gsr_shard_preprocess_p2p_raw_masked",
                       "gsr_sparse_preprocess_masked", "gsr_sparse_preprocess_raw_masked",
                       "gsr_shard_backward_render_masked", "gsr_shard_backward_preprocess_masked",
                       "gsr_shard_backward_preprocess_raw_masked", "gsr_sparse_backward_preprocess_masked",
                       "gsr_sparse_backward_preprocess_raw_masked")
# entry point -> (position of grad_mask, position of the camera or None) in its argument list
MASK_ARG = {"gsr_shard_preprocess_masked": (8, None), "gsr_shard_preprocess_raw_masked": (8, None),
            "gsr_shard_preprocess_p2p_masked": (10, None), "gsr_shard_preprocess_p2p_raw_masked": (10, None),
            "gsr_sparse_preprocess_masked": (9, None), "gsr_sparse_preprocess_raw_masked": (9, None),
            "gsr_shard_backward_preprocess_masked": (11, 10), "gsr_shard_backward_preprocess_raw_masked": (10, None),
            "gsr_sparse_backward_preprocess_masked": (13, 12), "gsr_sparse_backward_preprocess_raw_masked": (12, None)}


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
def test_entry_points_declared_exported_and_bound():
    lib = _lib.load()
    assert lib.gsr_abi_version() == 2
    header = open(_lib.os.path.join(_lib._HERE, "..", "include", "gsr_b200.h")).read()
    for name in MASKED_ENTRY_POINTS:
        assert name in _lib.SYMBOLS, name
        assert f"GSR_API int {name}(" in header, name
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and fn.argtypes, name


@pytest.mark.parametrize("name", sorted(MASK_ARG))
def test_entry_points_reject_a_null_mask_and_a_camera_before_the_device(name):
    lib = _lib.load()
    fn = getattr(lib, name)
    pos, cam_pos = MASK_ARG[name]
    args = [None] * len(fn.argtypes)
    for i, t in enumerate(fn.argtypes):   # every integer argument a plausible value, every pointer NULL
        if t in (C.c_int32, C.c_size_t):
            args[i] = 1
    assert fn(*args) == INVALID and b"grad_mask is null" in lib.gsr_last_error(), name
    if cam_pos is not None:
        args[pos] = C.c_void_p(256)
        cam = _lib.CameraGrads(C.c_void_p(256), C.c_void_p(256), C.c_void_p(256), C.c_void_p(256), 1 << 20)
        args[cam_pos] = C.byref(cam)
        assert fn(*args) == INVALID and b"camera" in lib.gsr_last_error(), name


def test_backward_render_masked_checks_its_scratch_before_the_device():
    lib = _lib.load()
    d = C.c_void_p(256)
    s = _lib.Settings(64, 64, 1.0, 1.0, 1.0, 0, 1, 0, 0, d, d, d, d)
    need = lib.gsr_grad_mask_scratch_bytes(64, 64)

    def call(mask_scratch=d, mbytes=need, owner=_lib.TileOwner(2, 1)):
        return lib.gsr_shard_backward_render_masked(C.byref(s), C.byref(owner), 100, 10, d, 1 << 20, d, 1 << 20, d,
                                                    1 << 20, d, None, None, d, 1 << 20, None, 0, mask_scratch, mbytes,
                                                    None)
    assert call(mask_scratch=None) == -3 and b"grad_mask scratch" in lib.gsr_last_error()
    assert call(mbytes=need - 1) == -3 and b"grad_mask scratch" in lib.gsr_last_error()
    assert call(owner=_lib.TileOwner(2, 2)) == INVALID and b"row_stride" in lib.gsr_last_error()


def _gloo_group():
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)


def test_forward_checks_the_mask_before_any_collective():
    if dist.is_initialized():
        pytest.skip("a process group already exists in this process")
    _gloo_group()
    try:
        cam = synth.ring_cameras(8, 4.5, 15.0, 64, 48, 61.0)[0]
        rs = settings_from(cam, (0.0, 0.0, 0.0), 0, "cpu")
        n = 10
        for camera_grad in (False, True):
            # the state forward reads before its first collective (the constructor's workspace queries need a GPU)
            rast = S.ShardedGaussianRasterizer.__new__(S.ShardedGaussianRasterizer)
            torch.nn.Module.__init__(rast)
            rast.raster_settings, rast.camera_grad, rast.deterministic = rs, camera_grad, False
            rast.exchange, rast.plan = S.Exchange(None), S.ShardPlan(n, 1, 0)

            def boom(*a, **k):
                raise AssertionError("a collective ran before the argument checks")
            for name in ("all_gather_inplace", "barrier", "all_reduce_sum", "reduce_scatter_sum",
                         "reduce_scatter_ordered", "broadcast", "all_to_all_single"):
                setattr(rast.exchange, name, boom)
            x = torch.zeros(n, 3)
            kw = dict(means3D=x, means2D=x, opacities=torch.zeros(n, 1), shs=torch.zeros(n, 1, 3), scales=x,
                      rotations=torch.zeros(n, 4))
            bad = [torch.zeros(n), torch.zeros(n, dtype=torch.int32), torch.zeros(n - 1, dtype=torch.bool),
                   torch.zeros(n + 1, dtype=torch.uint8), torch.zeros(n, 1, dtype=torch.bool),
                   torch.zeros(2 * n, dtype=torch.uint8)[::2], [1] * n]
            if camera_grad:
                bad.append(torch.ones(n, dtype=torch.bool))   # a good mask, but camera gradients sum over every Gaussian
            for m in bad:
                with pytest.raises(ValueError, match="grad_mask"):
                    rast(**kw, grad_mask=m)
            if not camera_grad:   # (forward_raw refuses a camera_grad module before it looks at the mask)
                with pytest.raises(ValueError, match="grad_mask"):
                    rast.forward_raw(x, x, torch.zeros(n, 1), torch.zeros(n, 1, 3), torch.zeros(n, 0, 3), x,
                                     torch.zeros(n, 4), grad_mask=torch.zeros(n - 1, dtype=torch.bool))
    finally:
        dist.destroy_process_group()


def test_sharded_edit_loop_rejects_an_unknown_grad_mask_mode():
    from gaussianeditor_b200.edit_loop import run_sharded_edit_loop
    with pytest.raises(ValueError, match="grad_mask"):
        run_sharded_edit_loop(steps=1, P=100, grad_mask="always")


# ---------------------------------------------------------------------------------------------------------------
# GPU: virtual ranks on one GPU
# ---------------------------------------------------------------------------------------------------------------
_CLOUD = {}


def _cloud():
    if not _CLOUD:
        cloud, _ = synth.make_config("c3", P=30011)   # not divisible by the world sizes: a padded tail
        _CLOUD["cloud"], _CLOUD["t"] = cloud, cloud_tensors(cloud, "cuda")
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


def _inputs(t, kind):
    """The per-Gaussian inputs of one form (full cloud), in shard_preprocess's order, plus features_rest for "raw"."""
    empty = torch.empty(0, device="cuda")
    P = t["means3D"].shape[0]
    if kind == "raw":
        op = t["opacities"].clamp(1e-4, 1 - 1e-4)
        return dict(args=(t["means3D"], t["shs"][:, :1].contiguous(), empty, torch.log(op / (1 - op)),
                          torch.log(t["scales"]), t["rotations"] * 1.7, empty), rest=t["shs"][:, 1:].contiguous())
    sh, colors, scales, rots, cov = t["shs"], empty, t["scales"], t["rotations"], empty
    if kind == "colors":
        sh, colors = empty, torch.rand(P, 3, generator=torch.Generator().manual_seed(5)).cuda()
    if kind == "cov":
        cov, scales, rots = _cov3d(t["scales"], t["rotations"]), empty, empty
    return dict(args=(t["means3D"], sh, colors, t["opacities"], scales, rots, cov), rest=None)


def _rank_args(inp, p):
    sl = lambda v: S.shard_slice(v, p) if v.numel() else v
    return tuple(sl(v) for v in inp["args"]), (None if inp["rest"] is None else sl(inp["rest"]))


def _rank_mask(mask, p):
    return None if mask is None else S.shard_slice(mask, p).contiguous().view(torch.uint8)


def _ordered_sum(parts):
    total = parts[0].clone()
    for q in parts[1:]:
        total += q
    return total


def _dense(world, rs, inp, dL, mask, det, depth=None, alpha=None, first_out=None):
    """Virtual dense ranks: (frame [4|5,H,W], radii [P_pad], per-slot gradients of the whole cloud)."""
    P = inp["args"][0].shape[0]
    H, W = rs.image_height, rs.image_width
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    geom = radii = None
    bufs = []
    for p in plans:
        args, rest = _rank_args(inp, p)
        b = S.shard_preprocess(p, rs, *args, geom=geom, radii=radii, raw_rest=rest, grad_mask=_rank_mask(mask, p))
        geom, radii = b.geom, b.radii
        bufs.append(b)
    for b in bufs:   # the all-gather: every rank holds every record
        b.geom = geom.clone(); b.radii = torch.full_like(radii, -7)
    planes = 4 if alpha is None else 5
    frame = torch.zeros(planes, H, W, device="cuda")
    accs = []
    for b in bufs:
        S.shard_order(b)
        part = torch.zeros(planes, H, W, device="cuda")
        S.shard_render(b, part[:3], part[3:4])
        if alpha is not None:
            S.shard_alpha(b, part[4:])
        frame += part
        if first_out is not None:
            first_out.append(_owner_first(b, dL))
        accs.append(S.shard_backward_render(b, dL, det, depth, alpha).clone())
    acc = _ordered_sum(accs)
    grads = [S.shard_backward_preprocess(b, acc[b.plan.base:b.plan.base + b.plan.slice_len].contiguous(),
                                         depth is not None) for b in bufs]
    return frame, bufs[0].radii.clone(), [torch.cat([g[i] for g in grads]) for i in range(len(grads[0]))]


def _sparse(world, rs, inp, dL, mask, det, depth=None):
    from gaussianeditor_b200 import sparse_sharded as SS
    P = inp["args"][0].shape[0]
    H, W = rs.image_height, rs.image_width
    ranks = [SS.SparseRank(S.ShardPlan(P, world, r), torch.device("cuda"), W, H) for r in range(world)]
    SS.link_virtual(ranks)
    for rk in ranks:
        rk.matrix.zero_()
    steps = []
    for rk in ranks:
        args, rest = _rank_args(inp, rk.plan)
        steps.append(SS.sparse_preprocess(rk, rs, *args, rk.cap_alloc, rest, _rank_mask(mask, rk.plan)))
    m = torch.stack([rk.matrix for rk in ranks]).sum(0)
    for rk in ranks:
        rk.matrix.copy_(m)
    for st in steps:
        SS.sparse_order(st)
    frame = torch.zeros(4, H, W, device="cuda")
    for st in steps:
        st.rk.frame.zero_()
        SS.sparse_render(st, st.rk.frame[:3], st.rk.frame[3:4])
        frame += st.rk.frame[:4]
    accs = [SS.sparse_backward_render(st, dL, det, depth) for st in steps]
    for st, acc in zip(steps, accs):
        SS.sparse_return(st, acc)
    grads = [SS.sparse_backward_preprocess(st, depth is not None) for st in steps]
    radii = torch.cat([rk.radii_local[:rk.plan.count] for rk in ranks])
    return frame, radii, [torch.cat([g[i] for g in grads]) for i in range(len(grads[0]))]


def _bits(t):
    return t.contiguous().view(torch.int32)


def _check_rows(masked, full, mask, exact):
    """Unedited rows +0.0 by bit pattern; edited rows equal `full` (bit for bit when `exact`, else rel L2 1e-5)."""
    assert len(masked) == len(full)
    for i, (g, f) in enumerate(zip(masked, full)):
        if g.numel() == 0:
            continue
        rows = g.reshape(g.shape[0], -1)
        assert not _bits(rows[~mask]).any(), f"slot {i}: an unedited row is not +0.0"
        if exact:
            assert torch.equal(_bits(rows[mask]), _bits(f.reshape(f.shape[0], -1)[mask])), f"slot {i}"
        elif mask.any():
            e = rel_l2(rows[mask].cpu().numpy(), f.reshape(f.shape[0], -1)[mask].cpu().numpy())
            assert e <= 1e-5, (i, e)


def _mask(kind, t, world, rs=None):
    P = t["means3D"].shape[0]
    if kind == "random30":
        return torch.rand(P, generator=torch.Generator().manual_seed(3)).cuda() < 0.3
    if kind == "spatial20":
        d = t["means3D"].norm(dim=1)
        return d <= d.kthvalue(max(1, int(0.2 * P))).values
    if kind == "all":
        return torch.ones(P, dtype=torch.bool, device="cuda")
    if kind == "none":
        return torch.zeros(P, dtype=torch.bool, device="cuda")
    if kind == "one_rank":   # the last rank's rows: every other tile owner supplies their gradients through the records
        p = S.ShardPlan(P, world, world - 1)
        m = torch.zeros(P, dtype=torch.bool, device="cuda")
        m[p.base:p.base + p.count] = True
        return m
    if kind == "culled":     # only Gaussians that are culled in this view: every gradient is zero
        from gaussianeditor_b200.rasterizer import GaussianRasterizer
        _, radii, _ = GaussianRasterizer(rs)(means3D=t["means3D"], means2D=torch.zeros_like(t["means3D"]),
                                             opacities=t["opacities"], shs=t["shs"], scales=t["scales"],
                                             rotations=t["rotations"])
        return radii == 0
    raise ValueError(kind)


def _single(rs, inp, dL, mask):
    """GaussianRasterizer(deterministic=True, grad_mask=mask): gradients in shard_backward_preprocess's slot order."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    args = [a.detach().clone().requires_grad_(True) if a.numel() else None for a in inp["args"]]
    m2 = torch.zeros_like(inp["args"][0], requires_grad=True)
    r = GaussianRasterizer(rs, deterministic=True, grad_mask=mask)
    color, _, _ = r(means3D=args[0], means2D=m2, shs=args[1], colors_precomp=args[2], opacities=args[3],
                    scales=args[4], rotations=args[5], cov3D_precomp=args[6])
    (color * dL).sum().backward()
    g = [a.grad if a is not None else None for a in args]
    return {"means3D": g[0], "means2D": m2.grad, "sh": g[1], "colors": g[2], "opacity": g[3], "scales": g[4],
            "rotations": g[5], "cov": g[6]}


def _camera(size, k=2):
    cam = synth.ring_cameras(8, 4.5, 15.0, size[0], size[1], 61.0)[k]
    return settings_from(cam, (0.2, 0.5, 0.1), 3, "cuda")


CASES = [  # world, mask, form, (W, H)
    (1, "random30", "sh", (400, 300)),
    (1, "all", "cov", (333, 201)),
    (2, "spatial20", "sh", (400, 300)),
    (2, "one_rank", "colors", (400, 300)),
    (3, "random30", "cov", (333, 201)),
    (3, "none", "sh", (333, 201)),
    (3, "culled", "sh", (400, 300)),
    (8, "one_rank", "sh", (400, 300)),
    (8, "spatial20", "colors", (64, 40)),    # 3 tile rows: five ranks own none
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,kind,form,size", CASES)
def test_virtual_ranks_masked_backward(world, kind, form, size):
    cloud, t = _cloud()
    rs = _camera(size)
    inp = _inputs(t, form)
    mask = _mask(kind, t, world, rs)
    dL = torch.rand(3, size[1], size[0], generator=torch.Generator().manual_seed(world)).cuda()
    f0, r0, full = _dense(world, rs, inp, dL, None, True)
    f1, r1, dense = _dense(world, rs, inp, dL, mask, True)
    assert torch.equal(_bits(f0), _bits(f1)) and torch.equal(r0, r1)   # the forward is unchanged
    _check_rows(dense, full, mask, exact=True)
    fs, _, sparse = _sparse(world, rs, inp, dL, mask, True)
    assert torch.equal(_bits(fs), _bits(f0[:4]))
    for a, b in zip(dense, sparse):                                     # dense equals sparse, bit for bit
        assert torch.equal(_bits(a), _bits(b))
    _, _, atomic = _dense(world, rs, inp, dL, mask, False)
    _check_rows(atomic, dense, mask, exact=False)
    _, _, atomic_sparse = _sparse(world, rs, inp, dL, mask, False)
    _check_rows(atomic_sparse, dense, mask, exact=False)
    if kind in ("none", "culled"):
        assert all(not _bits(g).any() for g in dense)
    if kind == "all":
        for a, b in zip(dense, full):
            assert torch.equal(_bits(a), _bits(b))
    if world == 1:   # the single-GPU masked rows
        ref = _single(rs, inp, dL, mask)
        order = ("means3D", "means2D", "sh", "colors", "opacity", "scales", "rotations", "cov")
        for name, g in zip(order, dense):
            if ref[name] is not None:
                assert torch.equal(_bits(g.reshape(ref[name].shape)), _bits(ref[name])), name


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 3])
@pytest.mark.parametrize("form", ["depth", "alpha", "raw", "raw_depth"])
def test_virtual_ranks_masked_forms(world, form):
    cloud, t = _cloud()
    size = (333, 201)
    rs = _camera(size)
    inp = _inputs(t, "raw" if form.startswith("raw") else "sh")
    mask = _mask("random30", t, world)
    g = torch.Generator().manual_seed(7)
    dL = torch.rand(3, size[1], size[0], generator=g).cuda()
    depth = torch.rand(1, size[1], size[0], generator=g).cuda() if form.endswith("depth") else None
    alpha = torch.rand(1, size[1], size[0], generator=g).cuda() if form == "alpha" else None
    f0, r0, full = _dense(world, rs, inp, dL, None, True, depth, alpha)
    f1, r1, dense = _dense(world, rs, inp, dL, mask, True, depth, alpha)
    assert torch.equal(_bits(f0), _bits(f1)) and torch.equal(r0, r1)
    _check_rows(dense, full, mask, exact=True)
    if alpha is None:
        _, _, sparse = _sparse(world, rs, inp, dL, mask, True, depth)
        for a, b in zip(dense, sparse):
            assert torch.equal(_bits(a), _bits(b))
    _, _, atomic = _dense(world, rs, inp, dL, mask, False, depth, alpha)
    _check_rows(atomic, dense, mask, exact=False)


def _layers(edited, per_layer=3000, seed=0):
    """Three overlapping layers at view depths 2, 4 and 6 over a 128x128 frame, interleaved in index; the mask selects
    layer `edited` (0 = front, 2 = back)."""
    rng = np.random.default_rng(seed)
    cam = synth._origin_camera(128, 128)
    xyz, layer = [], []
    for i, z in enumerate((2.0, 4.0, 6.0)):
        xyz.append(synth._at_pixels(cam, rng.uniform(-4, 132, per_layer), rng.uniform(-4, 132, per_layer),
                                    np.full(per_layer, z) + rng.uniform(-0.2, 0.2, per_layer)))
        layer.append(np.full(per_layer, i))
    perm = rng.permutation(3 * per_layer)
    xyz, layer = np.concatenate(xyz).astype(np.float32)[perm], np.concatenate(layer)[perm]
    P = xyz.shape[0]
    scales = (np.exp(rng.uniform(np.log(0.01), np.log(0.04), (P, 3))) * (xyz[:, 2:3] / 4.0)).astype(np.float32)
    q = rng.normal(size=(P, 4))
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    opac = rng.uniform(0.2, 0.7, (P, 1)).astype(np.float32)
    shs = rng.uniform(-0.5, 0.5, (P, 4, 3)).astype(np.float32)
    return synth.Cloud(xyz, scales, q, opac, shs, 1), cam, torch.from_numpy(layer == edited).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("edited", [0, 2])
def test_virtual_ranks_layered_scene(edited):
    cloud, cam, mask = _layers(edited)
    t = cloud_tensors(cloud, "cuda")
    rs = settings_from(cam, (0.0, 0.0, 0.0), cloud.sh_degree, "cuda")
    inp = _inputs(t, "sh")
    dL = torch.rand(3, 128, 128, generator=torch.Generator().manual_seed(1)).cuda()
    for world in (1, 3):
        _, _, full = _dense(world, rs, inp, dL, None, True)
        _, _, dense = _dense(world, rs, inp, dL, mask, True)
        _check_rows(dense, full, mask, exact=True)
        _, _, sparse = _sparse(world, rs, inp, dL, mask, True)
        for a, b in zip(dense, sparse):
            assert torch.equal(_bits(a), _bits(b))


def _owner_first(b, dL):
    """Runs the masked blend backward of buffer `b` (atomic) with first[] pre-filled with 0xAB bytes, and returns
    (first[] as uint32 numpy, ranges, n_contrib, point_list) for the restatement."""
    lib = _lib.load()
    W, H = b.W, b.H
    store = {}

    def get(name, n, dtype, grow):
        if name not in store:
            store[name] = torch.full((n,), 0xAB, dtype=torch.uint8, device="cuda") if name == "grad_mask_first" \
                else torch.empty(n, dtype=dtype, device="cuda")
        return store[name]
    acc = torch.empty(b.plan.P_pad, S.ACC_STRIDE, device="cuda")
    S.owner_backward_render(b.s, b.own, b.plan.P_pad, b.R, b.geom, b.binning, b.img, dL, acc, False, get, masked=True)
    torch.cuda.synchronize()
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)
    first = store["grad_mask_first"][:4 * ntiles].view(torch.int32).cpu().numpy().view(np.uint32)
    iv = _lib.ImageView()
    assert lib.gsr_view_image(S._ptr(b.img), W, H, C.byref(iv)) == 0
    ranges = S._view_bytes(b.img, iv.ranges, 8 * ntiles).view(torch.int32).cpu().numpy().view(np.uint32).reshape(-1, 2)
    nc = S._view_bytes(b.img, iv.n_contrib, 4 * W * H).view(torch.int32).cpu().numpy().view(np.uint32).reshape(H, W)
    pl = np.zeros(0, np.uint32)
    if b.R > 0:
        bv = _lib.BinningView()
        assert lib.gsr_view_binning(S._ptr(b.binning), b.plan.P_pad, b.R, W, H, C.byref(bv)) == 0
        pl = S._view_bytes(b.binning, bv.point_list, 4 * b.R).view(torch.int32).cpu().numpy().view(np.uint32)
    return b.plan, first, ranges, nc, pl


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_owner_first_matches_restatement(world):
    cloud, t = _cloud()
    size = (333, 201)
    rs = _camera(size)
    inp = _inputs(t, "sh")
    mask = _mask("spatial20", t, world)
    dL = torch.rand(3, size[1], size[0], generator=torch.Generator().manual_seed(2)).cuda()
    firsts = []
    _dense(world, rs, inp, dL, mask, True, first_out=firsts)
    P = t["means3D"].shape[0]
    gx, gy = (size[0] + 15) // 16, (size[1] + 15) // 16
    for plan, first, ranges, nc, pl in firsts:
        edited = np.zeros(plan.P_pad, bool)    # the global index space of the dense records
        m = mask.cpu().numpy()
        for r in range(world):
            p = S.ShardPlan(P, world, r)
            edited[p.base:p.base + p.count] = m[p.base:p.base + p.count]
        ncp = np.zeros((gy * 16, gx * 16), np.uint32)
        ncp[:nc.shape[0], :nc.shape[1]] = nc
        tile_last = ncp.reshape(gy, 16, gx, 16).max(axis=(1, 3)).reshape(-1)
        for tile in range(gx * gy):
            if (tile // gx) % world != plan.rank:
                assert first[tile] == 0xABABABAB, (plan.rank, tile)   # not owned: untouched
                continue
            x, y = ranges[tile]
            n = min(int(tile_last[tile]), int(y) - int(x)) if y > x else 0
            hit = np.nonzero(edited[pl[x:x + n]])[0]
            want = hit[0] + 1 if hit.size else 0xFFFFFFFF
            assert first[tile] == want, (plan.rank, tile)


# ---------------------------------------------------------------------------------------------------------------
# GPU: world 1 through a real NCCL group in this process
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nccl_world1():
    if dist.is_initialized():
        pytest.skip("a process group already exists in this process")
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1,
                            device_id=torch.device("cuda", 0))
    try:
        yield
    finally:
        dist.destroy_process_group()


MODULES = [dict(mode="dense", p2p=False), dict(mode="dense", p2p=True), dict(mode="sparse")]


def _module_grads(rast, inp, mask, dL, raw=False):
    args = [a.detach().clone().requires_grad_(True) if a.numel() else None for a in inp["args"]]
    m2 = torch.zeros_like(inp["args"][0], requires_grad=True)
    if raw:
        rest = inp["rest"].detach().clone().requires_grad_(True)
        color, radii, _ = rast.forward_raw(args[0], m2, args[3], args[1], rest, args[4], args[5], grad_mask=mask)
        leaves = [args[0], m2, args[3], args[1], rest, args[4], args[5]]
    else:
        color, radii, _ = rast(means3D=args[0], means2D=m2, shs=args[1], colors_precomp=args[2], opacities=args[3],
                               scales=args[4], rotations=args[5], cov3D_precomp=args[6], grad_mask=mask)
        leaves = [args[0], m2, args[1], args[2], args[3], args[4], args[5], args[6]]
    (color * dL).sum().backward()
    return color.detach(), radii, [a.grad if a is not None else torch.empty(0, device="cuda") for a in leaves]


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["sh", "raw"])
def test_world1_modes_agree_with_virtual_ranks(nccl_world1, form):
    cloud, t = _cloud()
    size = (400, 300)
    rs = _camera(size)
    inp = _inputs(t, form)
    mask = _mask("random30", t, 1)
    dL = torch.rand(3, size[1], size[0], generator=torch.Generator().manual_seed(4)).cuda()
    f_ref, _, ref = _dense(1, rs, inp, dL, mask, True)
    P = t["means3D"].shape[0]
    for kw in MODULES:
        rast = S.ShardedGaussianRasterizer(rs, P, deterministic=True, **kw)
        try:
            color, _, grads = _module_grads(rast, inp, mask, dL, raw=form == "raw")
        finally:
            rast.close()
        assert torch.equal(_bits(color), _bits(f_ref[:3])), kw
        for i, (a, b) in enumerate(zip(grads, ref)):
            if a.numel():   # the slots of the inputs in use
                assert torch.equal(_bits(a.reshape(b.shape)), _bits(b)), (kw, i)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["dense", "sparse"])
def test_world1_static_capacity_capture_and_overflow(nccl_world1, mode):
    cloud, t = _cloud()
    size = (400, 300)
    cams = [_camera(size, k) for k in (1, 2, 3)]
    inp = _inputs(t, "sh")
    P = t["means3D"].shape[0]
    mask = _mask("spatial20", t, 1)
    mbuf = torch.zeros(P, dtype=torch.bool, device="cuda")
    dL = torch.rand(3, size[1], size[0], generator=torch.Generator().manual_seed(6)).cuda()
    eager = []
    for rs in cams:
        _, _, g = _dense(1, rs, inp, dL, mask, True)
        eager.append(g)
    # exact capacity: R of the camera, read from an eager static forward of a generous module
    rast = S.ShardedGaussianRasterizer(cams[0], P, mode=mode, deterministic=True, static_capacity=1 << 22)
    try:
        _module_grads(rast, inp, mask, dL)
        R = rast.check_capacity()
    finally:
        rast.close()
    for cap, over in ((R, False), (R - 1, True)):
        rast = S.ShardedGaussianRasterizer(cams[0], P, mode=mode, deterministic=True, static_capacity=cap)
        try:
            color, _, g = _module_grads(rast, inp, mask, dL)
            if over:
                with pytest.raises(RuntimeError, match="static_capacity"):
                    rast.check_capacity()
                assert all(int(torch.count_nonzero(x)) == 0 for x in g)   # as the unmasked overflow: value zero
                for x in g:
                    if x.numel():
                        assert not _bits(x.reshape(P, -1)[~mask]).any()   # and the unedited rows +0.0
            else:
                assert rast.check_capacity() == R
                for a, b in zip(g, eager[0]):
                    if a.numel():
                        assert torch.equal(_bits(a.reshape(b.shape)), _bits(b))
        finally:
            rast.close()
    # a captured forward + backward with the mask, replayed for three cameras
    rast = S.ShardedGaussianRasterizer(cams[0], P, mode=mode, deterministic=True, static_capacity=1 << 22)
    try:
        leaves = [a.detach().clone().requires_grad_(True) if a.numel() else None for a in inp["args"]]
        m2 = torch.zeros_like(inp["args"][0], requires_grad=True)
        view, proj, campos = (cams[0].viewmatrix.clone(), cams[0].projmatrix.clone(), cams[0].campos.clone())
        rast.raster_settings = cams[0]._replace(viewmatrix=view, projmatrix=proj, campos=campos)
        mbuf.copy_(mask)

        def step():
            for a in leaves + [m2]:
                if a is not None:
                    a.grad = None
            color, _, _ = rast(means3D=leaves[0], means2D=m2, shs=leaves[1], opacities=leaves[3], scales=leaves[4],
                               rotations=leaves[5], grad_mask=mbuf)
            (color * dL).sum().backward()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                step()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        for a in leaves + [m2]:
            if a is not None:
                a.grad = None
        with torch.cuda.graph(graph):
            step()
        for k, rs in enumerate(cams):
            view.copy_(rs.viewmatrix); proj.copy_(rs.projmatrix); campos.copy_(rs.campos)
            graph.replay()
            torch.cuda.synchronize()
            got = [leaves[0].grad, m2.grad, leaves[1].grad, None, leaves[3].grad, leaves[4].grad, leaves[5].grad]
            for i, (a, b) in enumerate(zip(got, eager[k])):
                if a is not None and b.numel():
                    assert torch.equal(_bits(a.reshape(b.shape)), _bits(b)), (k, i)
    finally:
        rast.close()


@pytest.mark.gpu
def test_world1_sharded_edit_loop_kernel_equals_hooks(nccl_world1):
    from gaussianeditor_b200.edit_loop import run_sharded_edit_loop
    for mode in ("dense", "sparse"):
        kw = dict(steps=200, P=60000, densification_interval=100, seed=0, mode=mode, deterministic=True)
        a = run_sharded_edit_loop(grad_mask="hooks", **kw)
        b = run_sharded_edit_loop(grad_mask="kernel", **kw)
        assert len(a["densify"]) == 1 and len(set(a["counts"])) > 1, mode
        assert a["counts"] == b["counts"] and a["losses"] == b["losses"], mode
        for nm, p in a["params"].items():
            assert torch.equal(_bits(p), _bits(b["params"][nm])), (mode, nm)
        for ga, gb in zip(a["optimizer"].param_groups, b["optimizer"].param_groups):
            sa, sb = a["optimizer"].state[ga["params"][0]], b["optimizer"].state[gb["params"][0]]
            for key in ("exp_avg", "exp_avg_sq", "step"):
                assert torch.equal(sa[key], sb[key]), (mode, ga["name"], key)

