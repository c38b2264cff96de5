"""Binning, blending and tracing on the LIST STRUCTURES the binning and render kernels depend on (synth.hotspot_cloud,
synth.tied_depth_cloud, synth.one_tile_cloud):
  * a hot tile whose list holds ~70 000 instances: more than one sort tile (4096) carries a single digit through the
    decoupled look-back, more than 2^16 (n_contrib, 16-bit staging), every pixel walks the whole list and lists end at
    every position of render_bwd's four-splat batches and apply_weights' 256-splat rounds;
  * ~27 000 visible Gaussians on one depth key plus exact copies appended far away in index (densify_and_clone): equal
    keys must come out in Gaussian-index order inside every tile (the reference sorts `tile|depth` stably);
  * instance counts R == P at and next to the multiples of 32, 128, 512 and 4096, and the speculative forward's
    capacity test at cap = R - 1, R, R + 1.
CPU: the generators are seeded and hit those edges (CPU oracle). GPU: forward bit-exact against the reference's own
CUDA build (or its recorded digests, tests/golden/parity/reference_outputs.npz), backward against it and the fp64
oracle, deterministic mode, apply_weights and the Gaussian-sharded paths against one GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import _lib, synth
from oracle import cpu_oracle
from util import cloud_tensors, rel_l2, run_ours, settings_from

ONE_TILE_SPEC = (4095, 4096, 4097)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_list_generators_are_seeded_and_hit_their_edges():
    for gen in (synth.hotspot_cloud, synth.tied_depth_cloud, lambda: synth.one_tile_cloud(4097)):
        (a, _), (b, _) = gen(), gen()
        for k in ("means3D", "scales", "rotations", "opacities", "shs"):
            assert np.array_equal(getattr(a, k), getattr(b, k)), k
    # hot spot: one list longer than 2^16, n_contrib above 2^16, no pixel at the T < 1e-4 stop
    cloud, cam = synth.hotspot_cloud()
    f = cpu_oracle.forward_from(cloud, cam, colors_precomp=np.ones((cloud.means3D.shape[0], 3), np.float32))
    try:
        lens = f.ranges[:, 1].astype(np.int64) - f.ranges[:, 0]
        assert lens.max() > 65536 and f.n_contrib.max() > 65536, (lens.max(), f.n_contrib.max())
        assert f.final_T.min() > 1e-4 and np.count_nonzero(lens) == lens.size
    finally:
        f.close()
    # tied depths: >= 8192 visible Gaussians on one depth key, exact copies of earlier rows at the end
    cloud, cam = synth.tied_depth_cloud()
    f = cpu_oracle.forward_from(cloud, cam, render=False)
    try:
        vis = f.radii > 0
        _, ties = np.unique(f.depths[vis], return_counts=True)
        assert ties.max() >= 8192, ties.max()
        rows = np.concatenate([cloud.means3D, cloud.scales, cloud.rotations, cloud.opacities], 1)
        _, first = np.unique(rows, axis=0, return_index=True)
        copies = np.setdiff1d(np.arange(rows.shape[0]), first)
        assert copies.size > 0.3 * first.size and copies.min() >= first.size   # appended after every original
    finally:
        f.close()
    # one tile per Gaussian: R == P exactly, distinct depths
    for P in synth.ONE_TILE_COUNTS:
        cloud, cam = synth.one_tile_cloud(P)
        f = cpu_oracle.forward_from(cloud, cam, render=False)
        try:
            assert np.all(f.tiles_touched == 1) and f.num_rendered == P, P
            assert np.unique(f.depths).size == P
            if P >= 4096:
                assert (f.ranges[:, 1] - f.ranges[:, 0]).max() > 512     # a few long lists
        finally:
            f.close()


# ---------------------------------------------------------------------------------------------------------------- GPU
_SCENES = {}


def _scene(name):
    """(cloud, cam, bg) of a scene name: "hotspot", "tied_depth" or "one_tile/<P>"."""
    if name not in _SCENES:
        if name == "hotspot":
            cloud, cam = synth.hotspot_cloud()
            bg = (0.1, 0.2, 0.3)
        elif name == "tied_depth":
            cloud, cam = synth.tied_depth_cloud()
            bg = (0.3, 0.2, 0.1)
        else:
            cloud, cam = synth.one_tile_cloud(int(name.split("/")[1]))
            bg = (0.0, 0.5, 1.0)
        _SCENES.clear()
        _SCENES[name] = (cloud, cam, bg)
    return _SCENES[name]


def _dL(cam, seed=47):
    return np.random.default_rng(seed).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)


def _assert_lists_sorted_and_stable(views, R):
    """Inside every tile: depth keys ascending, equal keys in ascending Gaussian index. Returns the number of adjacent
    tied pairs inside a tile."""
    rng = views["ranges"].cpu().numpy().astype(np.int64)
    pl = views["point_list"].cpu().numpy().astype(np.int64)
    assert pl.size == R
    tile = np.zeros(R, np.int64)
    nz = rng[:, 1] > rng[:, 0]
    tile[rng[nz, 0]] = 1
    same = np.cumsum(tile)[1:] == np.cumsum(tile)[:-1]        # neighbours in the same tile's range
    d = views["records"][:, 6].cpu().numpy().view(np.uint32)[pl]
    assert np.all(d[1:][same] >= d[:-1][same])
    tie = same & (d[1:] == d[:-1])
    assert np.all(pl[1:][tie] > pl[:-1][tie])
    return int(tie.sum())


FWD_SCENES = ["hotspot", "tied_depth"] + [f"one_tile/{P}" for P in synth.ONE_TILE_COUNTS]


@pytest.mark.gpu
@pytest.mark.parametrize("scene", FWD_SCENES)
def test_forward_bit_exact_binning_and_depth_sort_variants(scene):
    """FWD_EXACT outputs bit-exact against the reference under both binning and both depth-sort variants (and every
    render_fwd variant on the hot spot and the tie layer); every tile's list depth-sorted with ties in index order."""
    from test_parity_gpu import FWD_EXACT, _options, _ours_forward_fields, _Ref, _ref_forward_fields, _ref_run
    cloud, cam, bg = _scene(scene)
    ref = _Ref(f"list_edges/{scene}/fwd", lambda: _ref_forward_fields(_ref_run(cloud, cam, bg)))
    for bv in (0, 1):
        for dv in (0, 1):
            with _options(binning_variant=bv, depth_sort_variant=dv):
                out = run_ours(cloud, cam, bg)
            fwd = _ours_forward_fields(out)
            bad = [k for k in FWD_EXACT if not ref.equal(k, fwd[k])]
            assert not bad, (scene, bv, dv, bad)
            ties = _assert_lists_sorted_and_stable(out["views"], out["R"])
            if scene == "tied_depth":
                assert ties >= 8192, ties
    if scene.startswith("one_tile"):
        assert out["R"] == cloud.means3D.shape[0]
    else:
        for v in range(6):
            with _options(render_fwd_variant=v):
                fwd = _ours_forward_fields(run_ours(cloud, cam, bg))
            bad = [k for k in FWD_EXACT if not ref.equal(k, fwd[k])]
            assert not bad, (scene, v, bad)
    if scene == "hotspot":
        assert int(fwd["n_contrib"].max()) > 65536 and float(fwd["final_T"].min()) > 1e-4


def _speculative(cloud, cam, bg, cap, guard=1 << 16):
    """Both forward halves through the C ABI with the second half launched for `cap` instances
    (gsr_forward_render_speculative) -> (R the device counted, forward state, colour, guard bytes behind the binning
    workspace untouched)."""
    import gaussianeditor_b200.rasterizer as RZ
    lib = _lib.load()
    dev = torch.device("cuda")
    ct = cloud_tensors(cloud, dev)
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    P, M, W, H = cloud.means3D.shape[0], cloud.shs.shape[1], cam.image_width, cam.image_height
    keep = []
    s = RZ._make_settings(rs, M, dev, keep)
    c = RZ._make_cloud(P, ct["means3D"], ct["opacities"], ct["shs"], None, ct["scales"], ct["rotations"], None)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    state = RZ._ForwardState()
    state.P, state.M, state.W, state.H = P, M, W, H
    state.radii = torch.empty(P, dtype=torch.int32, device=dev)
    gbytes = lib.gsr_geometry_bytes(P)
    state.geom = torch.empty(gbytes, dtype=torch.uint8, device=dev)
    pinned = torch.full((1,), -1, dtype=torch.int32).pin_memory()
    _lib.check(lib.gsr_forward_preprocess(C.byref(s), C.byref(c), RZ._ptr(state.geom), gbytes, RZ._ptr(state.radii),
                                          C.c_void_p(pinned.data_ptr()), st), "gsr_forward_preprocess")
    ibytes = lib.gsr_image_bytes(W, H)
    state.img = torch.empty(ibytes, dtype=torch.uint8, device=dev)
    bbytes = lib.gsr_binning_bytes(P, cap, W, H)
    buf = torch.full((bbytes + guard,), 0xA5, dtype=torch.uint8, device=dev)
    state.binning = buf[:bbytes]
    state.binning.zero_()      # a list the kernels leave unwritten then names Gaussian 0, never an index out of range
    color = torch.empty(3, H, W, device=dev)
    depth = torch.empty(1, H, W, device=dev)
    _lib.check(lib.gsr_forward_render_speculative(C.byref(s), C.byref(c), cap, RZ._ptr(state.geom), gbytes,
                                                  RZ._ptr(state.binning), bbytes, RZ._ptr(state.img), ibytes,
                                                  RZ._ptr(state.radii), RZ._ptr(color), RZ._ptr(depth), st),
               "gsr_forward_render_speculative")
    torch.cuda.synchronize()
    R = int(pinned[0])
    state.num_rendered, state.cap = R, cap
    return R, state, color, depth, bool((buf[bbytes:] == 0xA5).all())


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["hotspot"] + [f"one_tile/{P}" for P in ONE_TILE_SPEC])
def test_speculative_capacity_boundaries(scene):
    """The speculative second half at capacity R - 1 (must be seen as an overflow: the count exceeds the capacity, the
    ranges stay empty and nothing is written past the workspace) and at R and R + 1 (must give the exact path's
    point_list, ranges, n_contrib and images), under both binning variants."""
    import gaussianeditor_b200.rasterizer as RZ
    from test_parity_gpu import _options
    cloud, cam, bg = _scene(scene)
    for bv in (0, 1):
        with _options(binning_variant=bv):
            try:
                RZ.SPECULATIVE = False
                exact = run_ours(cloud, cam, bg)
            finally:
                RZ.SPECULATIVE = True
            R = exact["R"]
            ev = exact["views"]
            for cap in (R - 1, R, R + 1):
                got, state, color, depth, guard_ok = _speculative(cloud, cam, bg, cap)
                assert got == R and guard_ok, (scene, bv, cap)
                if cap < R:
                    if bv == 1:
                        assert int(RZ.forward_state_views(state)["ranges"].abs().sum()) == 0, (scene, cap)
                    continue
                v = RZ.forward_state_views(state)
                for k in ("point_list", "ranges", "n_contrib", "final_T"):
                    assert torch.equal(v[k], ev[k]), (scene, bv, cap, k)
                assert torch.equal(color, exact["color"]) and torch.equal(depth, exact["depth"]), (scene, bv, cap)


BWD_SCENES = ["hotspot", "tied_depth", "one_tile/33", "one_tile/4097"]


@pytest.mark.gpu
@pytest.mark.parametrize("scene", BWD_SCENES)
def test_backward_against_reference_and_fp64(scene):
    """All six gradients against the reference and the fp64 CPU oracle under render_bwd variants 15 (default: starts
    at the list's end and flushes four splats at a time, so lists of every length mod 4 end mid-batch), 14 and 0.
    Distance from fp64 at most 5e-5 as for the other edge scenes, except on the one-tile scenes (sub-pixel splats of
    opacity 0.2..0.9, one per tile list position): there the reference's own fp32 gradients are 5.4e-5 (dmean2D) and
    5.9e-5 / 7.1e-5 (dmean3D, P = 4097 / 33) from fp64, measured on an H100, and ours agree with them to the last
    digits, so the bound is 1e-4."""
    from test_parity_gpu import GRAD_PAIRS, _grads_vs_reference_and_truth, _options
    cloud, cam, bg = _scene(scene)
    dL = _dL(cam)
    truth_tol = 1e-4 if scene.startswith("one_tile") else 5e-5
    for v in (15, 14, 0):
        with _options(render_bwd_variant=v):
            ours = run_ours(cloud, cam, bg, dL=dL)
        _grads_vs_reference_and_truth(f"list_edges/{scene}/bwd", cloud, cam, bg, dL, ours, GRAD_PAIRS, truth_tol)


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["hotspot", "tied_depth"])
def test_deterministic_mode_repeatable_and_close(scene):
    """Deterministic backward (emission slots in depth order, ties included): same bits twice, within 1e-5 of the
    default backward."""
    from test_deterministic import _bits_equal, _grads
    cloud, cam, bg = _scene(scene)
    for mode in ("sh", "depth"):
        f1, g1 = _grads(cloud, cam, mode, True, bg=bg)
        f2, g2 = _grads(cloud, cam, mode, True, bg=bg)
        _bits_equal(g1, g2)
        _bits_equal(f1, f2)
        f0, g0 = _grads(cloud, cam, mode, False, bg=bg)
        _bits_equal(f0, f1)
        for k in g0:
            assert rel_l2(g1[k].numpy(), g0[k].numpy()) <= 1e-5, (scene, mode, k, rel_l2(g1[k].numpy(), g0[k].numpy()))


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["hotspot", "tied_depth"])
@pytest.mark.parametrize("CH", [1, 3])
def test_apply_weights_matches_reference(scene, CH):
    """apply_weights with binary masks: `cnt` and `weights` (sums of 0/1, exact in fp32) equal the reference's bit for
    bit, in the default and the deterministic form."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    from oracle import ref_cuda
    from test_parity_gpu import _Ref
    dev = "cuda"
    cloud, cam, _ = _scene(scene)
    H, W = cam.image_height, cam.image_width
    ct = cloud_tensors(cloud, dev)
    rs = settings_from(cam, (0, 0, 0), 0, dev)
    P = ct["means3D"].shape[0]
    mask = torch.from_numpy((np.random.default_rng(CH).uniform(size=(CH, H, W)) > 0.4).astype(np.float32)).to(dev)

    def compute():
        w = torch.zeros(P, CH, device=dev); c = torch.zeros(P, 1, dtype=torch.int32, device=dev)
        ref_cuda.ReferenceRasterizer().apply_weights(
            means3D=ct["means3D"], opacities=ct["opacities"], scales=ct["scales"], rotations=ct["rotations"], weights=w,
            cnt=c, image_weights=mask, bg=rs.bg, viewmatrix=rs.viewmatrix, projmatrix=rs.projmatrix, campos=rs.campos,
            tanfovx=rs.tanfovx, tanfovy=rs.tanfovy, image_height=H, image_width=W)
        torch.cuda.synchronize()
        return dict(cnt=c, cnt_sum=int(c.sum()), weights=w)
    ref = _Ref(f"list_edges/{scene}/apply_weights/{CH}", compute)
    assert ref.scalar("cnt_sum") > 0
    for det in (False, True):
        w = torch.zeros(P, CH, device=dev); c = torch.zeros(P, 1, dtype=torch.int32, device=dev)
        GaussianRasterizer(rs, deterministic=det).apply_weights(ct["means3D"], None, ct["opacities"], None, w,
                                                                ct["scales"], ct["rotations"], None, c, mask)
        torch.cuda.synchronize()
        assert ref.equal("cnt", c), (scene, CH, det)
        assert ref.equal("weights", w), (scene, CH, det)


SHARD_CASES = [("dense", 2, None), ("dense", 3, None), ("dense", 8, None), ("sparse", 2, "tight"),
               ("sparse", 3, "tight"), ("sparse", 8, "tight"), ("sparse", 2, "overflow"), ("sparse", 8, "overflow")]


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["hotspot", "tied_depth"])
@pytest.mark.parametrize("path,world,cap_mode", SHARD_CASES)
def test_sharded_virtual_ranks_match_single_gpu(scene, path, world, cap_mode):
    """The Gaussian-sharded rasterizer on virtual ranks (tests/test_sharded.py drivers): frames, depth and radii
    bit-identical to one GPU, the ranks' instance counts add up to R, gradients within 2e-5. On the hot spot every
    record goes to the one rank that owns tile row 1: the sparse exchange's largest segment holds nearly all of them,
    and `overflow` starts it at half that size."""
    from test_sharded import virtual_dense, virtual_sparse
    cloud, cam, bg = _scene(scene)
    dL = _dL(cam, seed=48)
    case = dict(cloud=cloud, cam=cam, bg=bg, dL=dL, ref=run_ours(cloud, cam, bg=bg, dL=dL))
    if path == "dense":
        virtual_dense(case, world)
    else:
        virtual_sparse(case, world, cap_mode)
