"""Tile binning over the whole supported tile grid (csrc/tile_binning.cu, the default path for gx * gy < 65536 tiles).

The tile-id bit length b = higher_msb(gx * gy) picks the kernels: pass 1 (which also emits the instances) sorts on
ceil(b / 2) bits and pass 2 on floor(b / 2) bits, each by its own instantiation tile_sort_pass_kernel<EMIT, NBITS>,
and at b = 1 pass 2 is a copy. So the frame size alone decides which of the 16 sort kernels run. Other switches
tied to the grid: tile_prefix_kernel keeps the 2-D prefix in shared memory while (gx + 1)(gy + 1) <= 10240 and uses
global scratch above; each of its threads walks ceil(gx gy / 1024) tiles (up to 64); tile_diff_copies goes from 64
replicas of the difference array down to 1; at 65536 tiles binning moves to the CUB path with 32-bit keys.

FRAMES has a frame for every b from 1 to 16, both sides of each switch, DCI 4K, the largest grid on tile binning with
and without partial last tiles, and frames one tile tall and one tile wide with b = 16. Each gets a seeded
synth.tile_grid_cloud: instances in every tile row and column, empty tiles, R over several 4096-instance sort tiles,
splats over hundreds of tiles along the long axis and depth keys tied across tiles.

CPU: higher_msb and tile_diff_copies restated, the table's coverage, the scenes' layout, and the numpy restatement of
the lists against the CPU oracle's.
GPU, on every frame with the shipped options:
  * R, ranges and point_list equal, bit for bit, the numpy restatement built from our radii, centres and depth keys;
    the forward (lists, radii, n_contrib, final_T, colour, depth, alpha) equals the reference's CUDA build, or the
    digests recorded from it in tests/golden/parity/tile_grid_reference.npz;
  * colour, colour + depth and colour + alpha gradients, default and deterministic, against the fp64 CPU oracle under
    a signed upstream; the deterministic backward gives the same bits twice;
  * apply_weights with sparse masks in multiples of 2^-8: default and deterministic bit for bit, and the CPU oracle
    where the hit counts agree;
  * the speculative forward at capacity R (hit) and R - 1 (miss), static capacity at R (the default result) and R - 1
    (an empty frame, zero gradients);
and on the largest grid and the one-tile-tall frame grad_mask, on those and the one-tile-wide frame the dense and
sparse sharded paths at world 2 and 3. A profiler pass checks that the table launches every sort instantiation.
"""
import os
import re

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import synth
from util import cloud_tensors, rel_l2, settings_from

BG = (0.3, 0.2, 0.1)
TILE = 16
SORT_TILE = 4096
PREFIX_SMEM = 10240          # tile_prefix_kernel's shared-memory array, in entries of the difference array
PREFIX_THREADS = 1024
MAX_TILE_DIFF = 4 * (2 * 65536 + 64)
WIDE = 1 << 17               # from this many pixels along an axis fp32 pixel coordinates lose ~0.01 px (see below)

# (W, H) -> why it is in the table
FRAMES = {
    (16, 16): "one tile: b = 1, pass 2 is a copy",
    (32, 16): "b = 2",
    (48, 32): "b = 3",
    (64, 48): "b = 4",
    (80, 64): "b = 5",
    (128, 112): "b = 6",
    (160, 160): "b = 7",
    (256, 208): "b = 8",
    (333, 201): "b = 9, partial last tile row and column",
    (512, 400): "b = 10",
    (640, 480): "b = 11",
    (960, 720): "b = 12",
    (1600, 1200): "b = 13",
    (1600, 1600): "b = 14, 10201 prefix entries: the last grid in shared memory",
    (1616, 1600): "b = 14, 10302 prefix entries: the first in global scratch",
    (2560, 1440): "b = 14, four replicas of the difference array",
    (3472, 2416): "217 x 151 = 32767 tiles: the highest b = 15",
    (4096, 2048): "32768 tiles: the lowest b = 16",
    (3840, 2400): "16:10 4K, b = 16",
    (4096, 2160): "DCI 4K, b = 16",
    (4073, 4105): "255 x 257 = 65535 tiles with a partial last tile row and column",
    (4080, 4112): "255 x 257 = 65535 tiles: the largest grid on tile binning",
    (600008, 13): "one tile tall, 37501 tiles, b = 16",
    (13, 600008): "one tile wide, 37501 tiles, b = 16",
    (4096, 4096): "65536 tiles: the first grid on the CUB path",
}
NAMES = [f"{w}x{h}" for w, h in FRAMES]
TALL, WIDE_FRAME, LARGEST = "600008x13", "13x600008", "4080x4112"


def _wh(name):
    return tuple(int(v) for v in name.split("x"))


def _grid(name):
    W, H = _wh(name)
    return (W + TILE - 1) // TILE, (H + TILE - 1) // TILE


# ---------------------------------------------------------------------------------------------------------------- CPU
def higher_msb(n):
    """csrc/tile_binning.cu: higher_msb, step for step (a binary search for the bit length of a 32-bit n)."""
    msb = step = 16
    while step > 1:
        step //= 2
        msb = msb + step if n >> msb else msb - step
    if n >> msb:
        msb += 1
    return msb


def tile_diff_copies(gx, gy):
    """csrc/common.cuh: tile_diff_copies."""
    nent, c = (gx + 1) * (gy + 1), 1
    while c < 64 and (2 * c + 1) * nent <= MAX_TILE_DIFF // 4:
        c *= 2
    return c


def tile_binning_supported(gx, gy):
    return gx * gy < 65536 and (gx + 1) * (gy + 1) <= MAX_TILE_DIFF


def sort_kernels(gx, gy):
    """The (EMIT, NBITS) sort instantiations run_tile_binning launches for the grid (none on the CUB path)."""
    if not tile_binning_supported(gx, gy):
        return set()
    b = higher_msb(gx * gy)
    b1, b2 = (b + 1) // 2, b // 2
    return {(True, b1)} | ({(False, b2)} if b2 else set())


def test_higher_msb_is_the_bit_length():
    for n in range(1, 65537):
        assert higher_msb(n) == n.bit_length(), n


def test_frame_table_reaches_every_switch():
    grids = {n: _grid(n) for n in NAMES}
    tb = {n: g for n, g in grids.items() if tile_binning_supported(*g)}
    bits = {n: higher_msb(gx * gy) for n, (gx, gy) in tb.items()}
    assert sorted(set(bits.values())) == list(range(1, 17))
    launched = set().union(*(sort_kernels(*g) for g in tb.values()))
    assert launched == {(e, n) for e in (True, False) for n in range(1, 9)}, sorted(launched)
    assert any(bits[n] == 1 for n in tb)                                   # the single-digit copy
    ntile = {n: gx * gy for n, (gx, gy) in grids.items()}
    for n, t in (("4096x2048", 32768), ("3472x2416", 32767), ("4080x4112", 65535), ("4073x4105", 65535),
                 ("4096x4096", 65536)):
        assert ntile[n] == t, n
    assert bits["4096x2048"] == 16 and bits["3472x2416"] == 15 and bits["4096x2160"] == 16
    assert max(ntile[n] for n in tb) == 65535 and "4096x4096" not in tb
    assert all(W % TILE and H % TILE for W, H in [_wh("4073x4105")])       # partial last row and column
    # the prefix's shared-memory switch, from both sides
    ent = {n: (gx + 1) * (gy + 1) for n, (gx, gy) in tb.items()}
    assert ent["1600x1600"] == 10201 <= PREFIX_SMEM < ent["1616x1600"] == 10302
    # every replica count of the difference array, and the prefix's tiles per thread from 1 to 64
    assert {tile_diff_copies(*g) for g in tb.values()} == {1, 2, 4, 8, 16, 32, 64}
    per = {-(-ntile[n] // PREFIX_THREADS) for n in tb}
    assert min(per) == 1 and max(per) == 64
    # one tile tall and one tile wide with b = 16: fewer tile rows (or columns) than sharded ranks
    assert grids[TALL][1] == 1 and grids[WIDE_FRAME][0] == 1 and bits[TALL] == bits[WIDE_FRAME] == 16


def restate_lists(means2D, radii, depth_bits, gx, gy):
    """The reference's binning in numpy: every visible Gaussian emits one instance per tile of its tile_rect (fp32
    arithmetic as in csrc/common.cuh), and the instances are ordered by (tile id, depth bits, Gaussian index).
    -> (tiles_touched [P], ranges [gx gy, 2], point_list [R])."""
    P = radii.shape[0]
    px, py = means2D[:, 0].astype(np.float32), means2D[:, 1].astype(np.float32)
    r = radii.astype(np.float32)
    t, one = np.float32(TILE), np.float32(1)
    lo = lambda p, n: np.clip(np.trunc((p - r) / t), 0, n).astype(np.int64)
    hi = lambda p, n: np.clip(np.trunc((((p + r) + t) - one) / t), 0, n).astype(np.int64)
    x0, x1, y0, y1 = lo(px, gx), hi(px, gx), lo(py, gy), hi(py, gy)
    cnt = np.where(radii > 0, (x1 - x0) * (y1 - y0), 0)
    g = np.repeat(np.arange(P), cnt)
    k = np.arange(g.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    w = (x1 - x0)[g]
    tile = (y0[g] + k // w) * gx + x0[g] + k % w
    order = np.lexsort((g, depth_bits[g].astype(np.int64), tile))
    tile, g = tile[order], g[order]
    ids = np.arange(gx * gy)
    first, last = np.searchsorted(tile, ids, "left"), np.searchsorted(tile, ids, "right")
    ranges = np.where((last > first)[:, None], np.stack([first, last], 1), 0)
    return cnt, ranges, g


_SCENES = {}


def _scene(name):
    if name not in _SCENES:
        _SCENES.clear()
        _SCENES[name] = synth.tile_grid_cloud(*_wh(name))
    return _SCENES[name]


def _check_layout(name, ranges, tiles_touched, depths, R):
    """The scene's promises on its forward: instances in every tile row and column, empty tiles where the grid has two
    or more of each and at least 50 tiles (on smaller grids the row and column splats and the fillers reach every tile), R over several sort tiles, a splat over hundreds of tiles along the long axis (or the whole
    axis where it is shorter), equal depth keys in different tiles."""
    gx, gy = _grid(name)
    n = (ranges[:, 1].astype(np.int64) - ranges[:, 0]).reshape(gy, gx)
    assert (n.sum(1) > 0).all() and (n.sum(0) > 0).all(), name
    if gx >= 2 and gy >= 2 and gx * gy >= 50:
        assert (n == 0).any(), name
    assert R > 3 * SORT_TILE, (name, R)
    assert tiles_touched.max() >= min(200, max(gx, gy) // 2), name
    vis = tiles_touched > 0
    _, ties = np.unique(depths[vis], return_counts=True)
    assert ties.max() >= 100, name


@pytest.mark.parametrize("name", NAMES)
def test_scene_layout_and_list_restatement(name):
    """On the CPU oracle's forward: the scene keeps its promises, and restate_lists gives the oracle's own lists (the
    reference's duplicateWithKeys, sort and identifyTileRanges) from its radii, centres and depths."""
    from oracle import cpu_oracle
    cloud, cam = _scene(name)
    f = cpu_oracle.forward_from(cloud, cam, render=False)
    try:
        gx, gy = _grid(name)
        tt, ranges, pl = restate_lists(f.means2D, f.radii, f.depths.view(np.uint32), gx, gy)
        assert np.array_equal(tt, f.tiles_touched) and pl.size == f.num_rendered
        assert np.array_equal(ranges, f.ranges) and np.array_equal(pl, f.point_list)
        _check_layout(name, f.ranges, f.tiles_touched.astype(np.int64), f.depths, f.num_rendered)
    finally:
        f.close()


# ---------------------------------------------------------------------------------------------------------------- GPU
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "parity", "tile_grid_reference.npz")


def _forward(cloud, cam):
    """Forward through GaussianRasterizer with the alpha image: (colour, radii, depth, alpha, forward-state views)."""
    from gaussianeditor_b200.rasterizer import GaussianRasterizer, _RasterizeGaussians, forward_state_views
    ct = cloud_tensors(cloud, "cuda")
    rs = settings_from(cam, BG, cloud.sh_degree, "cuda")
    col, radii, depth, alpha = GaussianRasterizer(rs, return_alpha=True)(
        means3D=ct["means3D"], means2D=torch.zeros_like(ct["means3D"]), opacities=ct["opacities"], shs=ct["shs"],
        scales=ct["scales"], rotations=ct["rotations"])
    state = _RasterizeGaussians.last_state
    return col, radii, depth, alpha, forward_state_views(state), int(state.num_rendered)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_lists_and_forward(name):
    """R, ranges and point_list bit for bit the numpy restatement from our own radii, centres and depth keys; every
    forward output bit for bit the reference's CUDA build."""
    from test_parity_gpu import _Ref, _ref_forward_fields, _ref_run
    cloud, cam = _scene(name)
    gx, gy = _grid(name)
    col, radii, depth, alpha, v, R = _forward(cloud, cam)
    rec = v["records"].cpu().numpy()
    rad = radii.cpu().numpy()
    tt, ranges, pl = restate_lists(rec[:, 0:2], rad, rec[:, 6].view(np.uint32), gx, gy)
    assert R == pl.size, (name, R, pl.size)
    assert np.array_equal(v["tiles_touched"].cpu().numpy().astype(np.int64), tt), name
    got_ranges = v["ranges"].cpu().numpy().astype(np.int64)
    bad = np.flatnonzero((got_ranges != ranges).any(1))
    assert bad.size == 0, (name, "ranges", bad[:8].tolist(), got_ranges[bad[:4]].tolist(), ranges[bad[:4]].tolist())
    got_pl = v["point_list"].cpu().numpy().astype(np.int64)
    bad = np.flatnonzero(got_pl != pl)
    assert bad.size == 0, (name, "point_list", bad.size, bad[:8].tolist())
    _check_layout(name, got_ranges, tt, rec[:, 6], R)

    def compute():
        ref = _ref_run(cloud, cam, BG)
        out = _ref_forward_fields(ref)
        out["alpha"] = 1.0 - ref["state"]["final_T"]
        return out
    ref = _Ref(f"tile_grid/{name}/fwd", compute, golden=GOLDEN)
    ours = dict(R=R, radii=radii, tiles_touched=v["tiles_touched"], ranges=v["ranges"], point_list=v["point_list"],
                n_contrib=v["n_contrib"], final_T=v["final_T"], color=col, depth=depth, alpha=alpha[0])
    bad = [k for k, x in ours.items() if not ref.equal(k, x)]
    assert not bad, (name, bad)


def _signed_upstreams(cam, seed):
    """Colour and depth upstreams uniform in [-1, 1): the gradient sums cancel, as a real loss's do."""
    rng = np.random.default_rng(seed)
    H, W = cam.image_height, cam.image_width
    return (rng.uniform(-1, 1, size=(3, H, W)).astype(np.float32),
            rng.uniform(-1, 1, size=(H, W)).astype(np.float32))


_SKIP = ("drot",)        # isotropic Gaussians: the rotation gradient is zero in exact arithmetic, rounding noise here
TRUTH_TOL = 5e-5
# Frames at least WIDE pixels along an axis: pixel coordinates near 6e5 carry an fp32 ulp of 1/16 px, and the
# gradients' fp32 differences (pixel - centre) lose ~0.01 px that the fp64 oracle keeps, so fp64 is no yardstick there.
# Those frames are checked against the fp32 CPU oracle (the reference's arithmetic) and the reference's CUDA build.
# Measured on an H100 80GB HBM3 (700 W): at most 4.2e-7 from the fp32 oracle, default and deterministic, all forms.
WIDE_TOL = 5e-6


def _is_wide(name):
    return max(_wh(name)) >= WIDE


def _own_distance(name, form, cloud, cam, gC, gD, truth, keys):
    """How far the reference's own arithmetic lands from fp64 on this case, per tensor: for the colour and alpha
    losses the reference's CUDA build (the alpha loss is the colour loss on the background (bg0 - 1, bg1, bg2), see
    test_deterministic_truth._truth; recorded when the build is absent), for the depth loss, which the reference cannot
    differentiate, the fp32 CPU oracle."""
    from test_deterministic_truth import _truth, _truth_errors
    from test_parity_gpu import GRAD_PAIRS, _Ref, _ref_run
    if form == "depth":
        t32 = _truth(cloud, cam, BG, form, gC, gD, f32=True)
        return _truth_errors({k: np.asarray(t32[k]) for k in keys}, truth, _SKIP)
    bg = BG if form == "colour" else (BG[0] - 1.0, BG[1], BG[2])
    pairs = [(a, b) for a, b in GRAD_PAIRS if a not in _SKIP]

    def compute():
        g = _ref_run(cloud, cam, bg, dL=gC)["grads"]
        return _truth_errors({a: g[b].cpu().numpy() for a, b in pairs}, truth, _SKIP)
    ref = _Ref(f"tile_grid/{name}/{form}/ref_err", compute, golden=GOLDEN)
    return {a: ref.scalar(a) for a, _ in pairs}


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["colour", "depth", "alpha"])
@pytest.mark.parametrize("name", NAMES)
def test_backward_against_truth(name, form):
    """Default and deterministic gradients of the colour, colour + depth and colour + alpha losses under a signed
    upstream, per tensor, against the fp64 CPU oracle to 5e-5, or, where the reference's own arithmetic lands farther
    from fp64 (_own_distance: deep stacks of splats and upstreams that cancel), to that distance plus 1e-5; on the frames
    at least WIDE pixels long against the fp32 CPU oracle to WIDE_TOL. The deterministic backward gives the same bits
    twice. Measured on an H100 80GB HBM3 (700 W): 193 of the 375 (frame, form, tensor) checks on fp64 frames are above
    5e-5, all in dscale, dmean3D, dmean2D and dopacity on frames from 64x48 up; the worst is dscale on 4073x4105 under
    the colour loss, 7.37e-4, and the reference's CUDA build is as far to three digits (every tensor within 3.5e-6 of
    its own distance)."""
    from test_deterministic_truth import _run, _truth, _truth_errors
    cloud, cam = _scene(name)
    gC, gD = _signed_upstreams(cam, 81)
    kw = dict(gD=gD if form == "depth" else None, gA=gC[0] if form == "alpha" else None)
    det, _ = _run(cloud, cam, BG, gC, deterministic=True, **kw)
    again, _ = _run(cloud, cam, BG, gC, deterministic=True, **kw)
    for k in det:
        assert np.array_equal(det[k].view(np.int32), again[k].view(np.int32)), (name, form, k)
    default, _ = _run(cloud, cam, BG, gC, deterministic=False, **kw)
    wide = _is_wide(name)
    truth = _truth(cloud, cam, BG, form, gC, gD, f32=wide)
    errs = {m: _truth_errors(g, truth, _SKIP) for m, g in (("default", default), ("deterministic", det))}
    if wide:
        bound = {k: WIDE_TOL for k in errs["default"]}
    else:
        own = _own_distance(name, form, cloud, cam, gC, gD, truth, errs["default"].keys())
        bound = {k: max(TRUTH_TOL, own[k] + 1e-5) for k in errs["default"]}
    print(name, form, "fp32" if wide else "fp64", {k: (f"{errs['default'][k]:.2e}", f"{errs['deterministic'][k]:.2e}",
                                                      f"bound {bound[k]:.2e}") for k in bound})
    bad = {(m, k): (e, bound[k]) for m, d in errs.items() for k, e in d.items() if not e <= bound[k]}
    assert not bad, (name, form, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in NAMES if _is_wide(n)])
def test_wide_backward_against_reference(name):
    """On the frames too long for the fp64 oracle: the default colour backward against the reference's CUDA build, to
    1e-4 + 10x the reference's run-to-run difference (its float atomics) per tensor."""
    from test_deterministic_truth import _run
    from test_parity_gpu import GRAD_PAIRS, _Ref, _ref_run
    cloud, cam = _scene(name)
    gC, _ = _signed_upstreams(cam, 81)
    got, _ = _run(cloud, cam, BG, gC, deterministic=False)
    pairs = [(a, b) for a, b in GRAD_PAIRS if a not in _SKIP]

    def compute():
        r1, r2 = _ref_run(cloud, cam, BG, dL=gC), _ref_run(cloud, cam, BG, dL=gC)
        out = {b: r1["grads"][b] for _, b in pairs}
        out.update({"noise/" + b: rel_l2(r2["grads"][b].cpu().numpy(), r1["grads"][b].cpu().numpy()) for _, b in pairs})
        return out
    ref = _Ref(f"tile_grid/{name}/bwd", compute, close=[b for _, b in pairs], golden=GOLDEN)
    for a, b in pairs:
        err = rel_l2(*ref.pair(b, got[a]))
        print(name, a, f"{err:.2e}", "noise", f"{ref.scalar('noise/' + b):.2e}")
        assert err <= 1e-4 + 10 * ref.scalar("noise/" + b), (name, a, err)


def _sparse_dyadic_mask(CH, H, W, seed):
    """Multiples of 2^-8 in [0, 63/256] on one pixel in 64, zero elsewhere: every partial sum of a Gaussian's weights
    is a multiple of 2^-8 below 2^16 even for the splats over millions of pixels, so exact in fp32 in any order."""
    rng = np.random.default_rng(seed)
    m = rng.integers(0, 64, size=(CH, H, W)) / 256.0
    return (m * (rng.uniform(size=(1, H, W)) < 1.0 / 64)).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_apply_weights_and_capacity(name):
    """apply_weights default and deterministic bit for bit, and the fp32 CPU oracle on every Gaussian whose hit count
    it shares; the speculative forward at capacity R and R - 1; static capacity at R and R - 1."""
    import gaussianeditor_b200.rasterizer as RZ
    from oracle import cpu_oracle
    from test_deterministic_truth import _aw_gpu
    from test_list_edges import _speculative
    from test_static_capacity import _run as static_run, _upstream
    from util import run_ours
    cloud, cam = _scene(name)
    H, W = cam.image_height, cam.image_width
    P = cloud.means3D.shape[0]
    CH = 1 + NAMES.index(name) % 3
    mask = _sparse_dyadic_mask(CH, H, W, seed=91 + CH)
    w0, c0 = _aw_gpu(cloud, cam, mask, False)
    assert float(w0.max()) < 1 << 16 and int((c0 > 0).sum()) > 0
    w1, c1 = _aw_gpu(cloud, cam, mask, True)
    assert torch.equal(c0, c1) and torch.equal(w0.view(torch.int32), w1.view(torch.int32)), name
    f = cpu_oracle.forward_from(cloud, cam, colors_precomp=np.ones((P, 3), np.float32))
    try:
        wo, co = np.zeros((P, CH), np.float32), np.zeros((P, 1), np.int32)
        f.apply_weights(wo, co, mask)
    finally:
        f.close()
    same = (co == c0.numpy())[:, 0]
    assert (~same).mean() <= 1e-4, (name, int((~same).sum()))
    assert np.array_equal(w0.numpy()[same].view(np.int32), wo[same].view(np.int32)), name
    del mask
    # speculative forward: capacity R is a hit and gives the exact path's lists and images, R - 1 a detected miss
    try:
        RZ.SPECULATIVE = False
        exact = run_ours(cloud, cam, BG)
    finally:
        RZ.SPECULATIVE = True
    R = exact["R"]
    got, state, color, depth, guard_ok = _speculative(cloud, cam, BG, R)
    assert got == R and guard_ok, name
    v = RZ.forward_state_views(state)
    for k in ("point_list", "ranges", "n_contrib", "final_T"):
        assert torch.equal(v[k], exact["views"][k]), (name, k)
    assert torch.equal(color, exact["color"]) and torch.equal(depth, exact["depth"]), name
    got, state, _, _, guard_ok = _speculative(cloud, cam, BG, R - 1)
    assert got == R and guard_ok, name
    if tile_binning_supported(*_grid(name)):    # tile_prefix_kernel leaves every range empty on a miss
        assert int(RZ.forward_state_views(state)["ranges"].abs().sum()) == 0, name
    del exact, state, v, color, depth
    # static capacity: at R the default result with status [R, 0], at R - 1 an empty frame and zero gradients
    dev = torch.device("cuda")
    rs = settings_from(cam, BG, cloud.sh_degree, dev)
    up = _upstream(cam, dev)
    ref_out, ref_g, _ = static_run(rs, cloud, False, (), True, None, dev, up)
    out, g, rast = static_run(rs, cloud, False, (), True, R, dev, up)
    assert rast.status.tolist() == [R, 0], name
    assert all(torch.equal(a, b) for a, b in zip(out, ref_out)), name
    assert all(torch.equal(a, b) for a, b in zip(g, ref_g)), name
    out, g, rast = static_run(rs, cloud, False, (), True, R - 1, dev, up)
    assert rast.status.tolist() == [R, 1], name
    bgimg = torch.tensor(BG, dtype=torch.float32, device=dev)[:, None, None].expand(3, H, W)
    assert torch.equal(out[0], bgimg) and int(torch.count_nonzero(out[2])) == 0, name
    assert all(int(torch.count_nonzero(x)) == 0 for x in g), name


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sh", "depth"])
@pytest.mark.parametrize("name", [LARGEST, TALL])
def test_grad_mask(name, mode):
    """grad_mask (deterministic) on the largest grid and the one-tile-tall frame: edited rows equal the unmasked
    deterministic gradients bit for bit, the others are +0.0, the forward is unchanged."""
    from test_grad_mask import _check_masked
    cloud, cam = _scene(name)
    m = np.random.default_rng(5).uniform(size=cloud.means3D.shape[0]) < 0.3
    _check_masked(cloud, cam, mode, torch.from_numpy(m).cuda())


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name", [TALL, WIDE_FRAME, LARGEST])
def test_sharded_paths(name, world):
    """Dense and sparse virtual ranks (test_sharded's harness) on grids with fewer tile rows than ranks, one tile
    column, and 65535 tiles: frames, depth, radii and the instance total bit for bit the single GPU's, gradients to
    summation order."""
    from test_sharded import virtual_dense, virtual_sparse
    from util import run_ours
    cloud, cam = _scene(name)
    gC, _ = _signed_upstreams(cam, 83)
    case = dict(cloud=cloud, cam=cam, bg=BG, dL=gC, ref=run_ours(cloud, cam, bg=BG, dL=gC))
    virtual_dense(case, world, skip=_SKIP)
    virtual_sparse(case, world, "tight", max_fill=1.0, skip=_SKIP)   # one tile row: every record goes to one rank


_SORT = re.compile(r"tile_sort_pass_kernel<(true|false), (\d)>")


@pytest.mark.gpu
def test_table_launches_every_sort_kernel():
    """One forward per frame under torch.profiler: each frame launches the sort instantiations its bit length picks
    (sort_kernels) and tile_prefix_kernel, and nothing of the CUB path; the 65536-tile frame the CUB path and no tile
    sort. Over the table: all 16 instantiations, and tile_prefix_kernel with its sum in shared memory and in global
    scratch."""
    from torch.profiler import ProfilerActivity, profile
    seen, prefix_entries = set(), set()
    for name in NAMES:
        cloud, cam = _scene(name)
        _forward(cloud, cam)              # module loading and workspace sizing outside the profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _forward(cloud, cam)
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
        sorts = {(m.group(1) == "true", int(m.group(2))) for n in names for m in [_SORT.search(n)] if m}
        gx, gy = _grid(name)
        prefix = any("tile_prefix_kernel" in n for n in names)
        cub = any("emit_instances_kernel" in n for n in names) and any("DeviceRadixSort" in n for n in names)
        if tile_binning_supported(gx, gy):
            assert sorts == sort_kernels(gx, gy) and prefix and not cub, (name, sorts, prefix, cub)
            prefix_entries.add((gx + 1) * (gy + 1))
        else:
            assert not sorts and not prefix and cub, (name, sorts, prefix, cub)
        seen |= sorts
    print("sort instantiations launched:", sorted(seen))
    assert seen == {(e, n) for e in (True, False) for n in range(1, 9)}, sorted(seen)
    assert min(prefix_entries) <= PREFIX_SMEM < max(prefix_entries)
