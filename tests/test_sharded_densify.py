"""Densify / prune of a Gaussian-sharded cloud (gaussianeditor_b200/shard_rebalance.py): the rebalance plan, the row
moves with their Adam state under gloo, the global top-k, and on the GPU the rebalanced cloud's renders, the
rasterizer's re-creation at new sizes and the whole sharded edit loop against its single-GPU restatement."""
import gc
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from gaussianeditor_b200 import optim_surgery
from gaussianeditor_b200 import shard_rebalance as SR
from gaussianeditor_b200 import sharded as S


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


# ---------------------------------------------------------------------------------------------------------------
# rebalance_plan
# ---------------------------------------------------------------------------------------------------------------
def _replay(counts):
    """Check one count matrix: split sums, destination sizes, and that the pieces put every row at its position in the
    segment-major, rank-minor global order (computed here independently)."""
    counts = [list(map(int, row)) for row in counts]
    G, K = len(counts), len(counts[0])
    rb = SR.rebalance_plan(torch.tensor(counts), G)
    P_new = sum(map(sum, counts))
    assert all(p == S.ShardPlan(P_new, G, d) for d, p in enumerate(rb.plans))
    # label = global position of each local row
    order = [(k, r, j) for k in range(K) for r in range(G) for j in range(counts[r][k])]
    pos = {key: i for i, key in enumerate(order)}
    labels = []
    for r in range(G):
        labels.append(torch.tensor([pos[k, r, j] for k in range(K) for j in range(counts[r][k])], dtype=torch.int64))
    for r in range(G):
        assert sum(rb.splits[r]) == sum(counts[r])
    new = []
    for d in range(G):
        assert sum(rb.splits[r][d] for r in range(G)) == rb.plans[d].count
        chunks = []
        for r in range(G):
            sent = labels[r][rb.send_index(r)]
            off = sum(rb.splits[r][:d])
            chunks.append(sent[off:off + rb.splits[r][d]])
        recv = torch.cat(chunks)
        assert len(rb.pieces[d]) <= G * K
        new.append(recv[rb.recv_index(d)])
    assert torch.equal(torch.cat(new), torch.arange(P_new))
    return rb


@pytest.mark.parametrize("G", [1, 2, 3, 8])
@pytest.mark.parametrize("K", [1, 2, 3])
def test_rebalance_plan_random_counts(G, K):
    rng = np.random.default_rng(100 * G + K)
    for _ in range(12):
        hi = int(rng.choice([2, 7, 40, 300]))
        counts = rng.integers(0, hi, size=(G, K))
        if counts.sum() == 0:
            counts[0, 0] = 1
        _replay(counts)


@pytest.mark.parametrize("counts", [
    [[0, 0], [5, 2], [0, 0]],            # ranks with zero rows (before and after)
    [[1, 0], [0, 1], [0, 0], [0, 0]],    # P_new < world
    [[0], [0], [0], [1]],
    [[9, 0], [0, 0], [4, 3]],            # a rank whose whole slice was pruned
    [[0, 0, 0], [3, 1, 1], [0, 0, 0]],
    [[17, 2, 2], [0, 5, 5], [30, 0, 0]],
])
def test_rebalance_plan_edge_cases(counts):
    _replay(counts)


def test_rebalance_plan_rejects_an_empty_cloud_and_bad_matrices():
    with pytest.raises(ValueError):
        SR.rebalance_plan([[0, 0], [0, 0]], 2)
    with pytest.raises(ValueError):
        SR.rebalance_plan([[1, -1], [3, 0]], 2)
    with pytest.raises(ValueError):
        SR.rebalance_plan([[1, 2]], 2)


def test_pack_unpack_round_trip_is_bit_exact():
    g = torch.Generator().manual_seed(0)
    ts = [torch.randn(11, 3, generator=g), torch.randn(11, 0, 3), torch.rand(11, generator=g) > 0.5,
          torch.randint(-2 ** 62, 2 ** 62, (11, 2), generator=g), torch.randn(11, 15, 3, generator=g).double()]
    ts[0][3] = float("nan")
    idx = torch.tensor([4, 0, 10, 3, 3])
    out = SR.unpack_rows(SR.pack_rows(ts, idx), [SR.row_spec(t) for t in ts])
    for a, b in zip(out, ts):
        assert a.dtype == b.dtype and a.shape == (5,) + b.shape[1:]
        if b.numel():   # compared as bytes: NaN rows included
            assert torch.equal(a.view(torch.uint8), b[idx].contiguous().view(torch.uint8))


# ---------------------------------------------------------------------------------------------------------------
# rebalance under gloo, against the single-process restatement
# ---------------------------------------------------------------------------------------------------------------
NAMES = [("xyz", (3,)), ("f_rest", (15, 3)), ("opacity", (1,))]


def _full_cloud(P):
    """A CPU cloud with an Adam that has stepped twice (non-zero moments), a bool mask and an int64 generation."""
    g = torch.Generator().manual_seed(7)
    params = {n: nn.Parameter(torch.randn((P,) + s, generator=g)) for n, s in NAMES}
    opt = torch.optim.Adam([{"params": [p], "lr": 0.01, "name": n} for n, p in params.items()], eps=1e-15)
    for _ in range(2):
        for p in params.values():
            p.grad = torch.randn(p.shape, generator=g)
        opt.step()
    mask = torch.rand(P, generator=g) > 0.6
    gen = torch.arange(P, dtype=torch.int64) * 1000003 - 7
    keep = torch.rand(P, generator=g) > 0.3
    sel = (torch.rand(P, generator=g) > 0.8) & keep
    return opt, mask, gen, keep, sel


def _local_optimizer(full_opt, plan):
    groups, state = [], {}
    for grp in full_opt.param_groups:
        p = grp["params"][0]
        q = nn.Parameter(S.shard_slice(p.detach(), plan).clone())
        groups.append({"params": [q], "lr": grp["lr"], "name": grp["name"]})
        st = full_opt.state[p]
        state[q] = {k: (S.shard_slice(v, plan).clone() if v.dim() > 0 else v.clone()) for k, v in st.items()}
    opt = torch.optim.Adam(groups, eps=1e-15)
    for q, st in state.items():
        opt.state[q] = st
    return opt


def _densify(opt, mask, gen, keep, sel, K):
    """prune to `keep`, then append K-1 copies of the `sel` rows (copy c scaled by 0.5**c); returns (mask, gen, counts)"""
    kept = optim_surgery.prune_optimizer(opt, keep)
    clone = sel[keep]
    masks, gens, counts = [mask[keep]], [gen[keep]], [int(keep.sum())]
    for c in range(1, K):
        optim_surgery.cat_tensors_to_optimizer(opt, {n: p.detach()[clone] * 0.5 ** c for n, p in kept.items()})
        masks.append(mask[sel]); gens.append(gen[sel] + c); counts.append(int(sel.sum()))
    return torch.cat(masks), torch.cat(gens), counts


def _rebalance_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    res = {}
    try:
        ex = S.Exchange()
        P = 101
        for K in (2, 3):
            full_opt, mask, gen, keep, sel = _full_cloud(P)
            plan = S.ShardPlan(P, world, rank)
            opt = _local_optimizer(full_opt, plan)
            sl = lambda t: S.shard_slice(t, plan)
            lmask, lgen, counts = _densify(opt, sl(mask), sl(gen), sl(keep), sl(sel), K)
            steps = [opt.state[g["params"][0]]["step"].clone() for g in opt.param_groups]
            stats = {}
            new_plan, (nmask, ngen) = SR.rebalance(ex, plan, counts, opt, extras=(lmask, lgen), stats=stats)
            # the single-process restatement on the whole cloud
            fmask, fgen, _ = _densify(full_opt, mask, gen, keep, sel, K)
            ok = new_plan == S.ShardPlan(fmask.numel(), world, rank)
            ok = ok and torch.equal(nmask, S.shard_slice(fmask, new_plan)) and nmask.dtype == torch.bool
            ok = ok and torch.equal(ngen, S.shard_slice(fgen, new_plan)) and ngen.dtype == torch.int64
            for g, fg, st0 in zip(opt.param_groups, full_opt.param_groups, steps):
                p, fp = g["params"][0], fg["params"][0]
                ok = ok and isinstance(p, nn.Parameter) and torch.equal(p.detach(), S.shard_slice(fp.detach(), new_plan))
                for key in ("exp_avg", "exp_avg_sq"):
                    ok = ok and torch.equal(opt.state[p][key], S.shard_slice(full_opt.state[fp][key], new_plan))
                ok = ok and torch.equal(opt.state[p]["step"], st0) and torch.equal(st0, full_opt.state[fp]["step"])
            res[K] = (bool(ok), stats["row_bytes"])
        # malformed input on the last rank only: every rank raises ValueError, nobody hangs
        plan = S.ShardPlan(10, world, rank)
        x = torch.zeros(plan.count + (1 if rank == world - 1 else 0), 2)
        try:
            SR.rebalance(ex, plan, [plan.count], None, extras=(x,))
            res["bad"] = None
        except ValueError as e:
            res["bad"] = str(e)
        # an empty new cloud raises everywhere too
        try:
            SR.rebalance(ex, plan, [0], None, extras=(torch.zeros(0, 2),))
            res["empty"] = None
        except ValueError as e:
            res["empty"] = str(e)
    except Exception:
        res["error"] = traceback.format_exc()
    finally:
        out[rank] = res
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_rebalance_matches_single_process_densify(world):
    out = mp.Manager().dict()
    mp.spawn(_rebalance_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    msgs = set()
    for r in range(world):
        res = out[r]
        assert "error" not in res, res.get("error")
        row_bytes = 4 * (3 + 45 + 1) * 3 + 1 + 8     # params + exp_avg + exp_avg_sq, mask, generation
        assert res[2] == (True, row_bytes) and res[3] == (True, row_bytes), r
        assert res["bad"] is not None and f"rank {world - 1}" in res["bad"]
        assert res["empty"] is not None and "empty" in res["empty"]
        msgs.add(res["bad"])
    assert len(msgs) == 1   # the same error on every rank


# ---------------------------------------------------------------------------------------------------------------
# global_top_k under gloo
# ---------------------------------------------------------------------------------------------------------------
def _tie_values(P):
    g = torch.Generator().manual_seed(3)
    v = torch.randint(0, 4, (P,), generator=g).float()
    v[torch.rand(P, generator=g) > 0.8] = float("nan")      # NaN counts as 0
    return v


def _top_k_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    res = {}
    try:
        ex = S.Exchange()
        for P in (5, 61, 200):
            v = _tie_values(P)
            plan = S.ShardPlan(P, world, rank)
            for k in sorted({1, 2, P // 3, P // 2, P - 1, P} - {0}):
                res[P, k] = SR.global_top_k(ex, plan, S.shard_slice(v, plan), k)
        try:
            plan = S.ShardPlan(8, world, rank)
            SR.global_top_k(ex, plan, torch.zeros(plan.count + (rank == 0)), 2)
            res["bad"] = False
        except ValueError:
            res["bad"] = True
    except Exception:
        res["error"] = traceback.format_exc()
    finally:
        out[rank] = res
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_global_top_k_selects_exactly_k_with_ties(world):
    out = mp.Manager().dict()
    mp.spawn(_top_k_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    for r in range(world):
        assert "error" not in out[r], out[r].get("error")
        assert out[r]["bad"] is True
    for (P, k) in [key for key in out[0] if isinstance(key, tuple)]:
        got = torch.cat([out[r][P, k] for r in range(world)])
        v = torch.nan_to_num(_tie_values(P), nan=0.0)
        # independent rule: sort by (value descending, index ascending), first k
        want = torch.zeros(P, dtype=torch.bool)
        want[sorted(range(P), key=lambda i: (-float(v[i]), i))[:k]] = True
        assert int(got.sum()) == k and torch.equal(got, want), (P, k)
        assert torch.equal(SR.top_k_mask(_tie_values(P), k), want)


# ---------------------------------------------------------------------------------------------------------------
# GPU: virtual ranks
# ---------------------------------------------------------------------------------------------------------------
def _cloud_of(t, sh_degree):
    from gaussianeditor_b200 import synth
    n = lambda x: x.detach().cpu().numpy().copy()
    return synth.Cloud(means3D=n(t["means3D"]), scales=n(t["scales"]), rotations=n(t["rotations"]),
                       opacities=n(t["opacities"]), shs=n(t["shs"]), sh_degree=sh_degree)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 8])
def test_virtual_ranks_rebalanced_cloud_renders_as_one_gpu(world):
    """pack -> in-process exchange -> unpack on CUDA tensors for `world` virtual ranks; the rebalanced cloud equals the
    restated densify bit for bit, and its dense and sparse sharded renders equal GaussianRasterizer's."""
    from gaussianeditor_b200 import synth
    from test_sharded import virtual_dense, virtual_sparse
    from util import cloud_tensors, run_ours
    dev = torch.device("cuda")
    cloud, cams = synth.make_config("c3", P=60013)
    full = cloud_tensors(cloud, dev)
    P = cloud.means3D.shape[0]
    g = torch.Generator(device=dev).manual_seed(world)
    keep = torch.rand(P, generator=g, device=dev) > 0.25
    if world == 8:
        keep[S.ShardPlan(P, world, 5).base:S.ShardPlan(P, world, 5).base + S.ShardPlan(P, world, 5).count] = False
    sel = (torch.rand(P, generator=g, device=dev) > 0.9) & keep
    names = list(full)
    plans = [S.ShardPlan(P, world, r) for r in range(world)]
    local, counts = [], []
    for p in plans:
        k, s = S.shard_slice(keep, p), S.shard_slice(sel, p)
        local.append([torch.cat((S.shard_slice(full[n], p)[k], S.shard_slice(full[n], p)[s])) for n in names])
        counts.append([int(k.sum()), int(s.sum())])
    rb = SR.rebalance_plan(counts, world)
    specs = [SR.row_spec(t) for t in local[0]]
    sends = [SR.pack_rows(local[r], rb.send_index(r, dev)) for r in range(world)]
    slices = []
    for d in range(world):
        recv = torch.cat([sends[r][sum(rb.splits[r][:d]):sum(rb.splits[r][:d + 1])] for r in range(world)])
        slices.append(SR.unpack_rows(recv.index_select(0, rb.recv_index(d, dev)), specs))
    new = {n: torch.cat([s[i] for s in slices]) for i, n in enumerate(names)}
    for n in names:
        assert torch.equal(new[n], torch.cat((full[n][keep], full[n][sel]))), n
    moved = _cloud_of(new, cloud.sh_degree)
    cam = cams[0]
    bg = (0.2, 0.5, 0.1)
    dL = np.random.default_rng(3).random((3, cam.image_height, cam.image_width), dtype=np.float32)
    case = dict(cloud=moved, cam=cam, bg=bg, dL=dL, ref=run_ours(moved, cam, bg=bg, dL=dL))
    virtual_dense(case, world)
    virtual_sparse(case, world, "full")


# ---------------------------------------------------------------------------------------------------------------
# GPU: world 1 in this process (NCCL)
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


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["dense", "sparse"])
def test_rasterizer_recreated_at_new_sizes_is_single_gpu_exact_and_frees_its_memory(nccl_world1, mode):
    from gaussianeditor_b200 import _lib, synth
    from gaussianeditor_b200 import sparse_sharded as SS
    from gaussianeditor_b200.rasterizer import GaussianRasterizer, _geometry_bytes
    from util import cloud_tensors, settings_from
    dev = torch.device("cuda", 0)
    cloud, cams = synth.make_config("c3", P=40000)
    cam = cams[1]
    rs = settings_from(cam, (0.1, 0.2, 0.3), cloud.sh_degree, dev)
    full = cloud_tensors(cloud, dev)
    sizes = [40000, 25007, 33333]

    def cycle(P):
        t = {n: v[:P] for n, v in full.items()}
        ref_c, ref_r, ref_d = GaussianRasterizer(rs, deterministic=True)(
            means3D=t["means3D"], means2D=torch.zeros_like(t["means3D"]), opacities=t["opacities"], shs=t["shs"],
            scales=t["scales"], rotations=t["rotations"])
        rast = S.ShardedGaussianRasterizer(rs, P, mode=mode, deterministic=True)
        assert rast.mode == mode and rast.plan.P_total == P
        with torch.no_grad():
            c, r, d = rast(means3D=t["means3D"], means2D=torch.zeros_like(t["means3D"]), opacities=t["opacities"],
                           shs=t["shs"], scales=t["scales"], rotations=t["rotations"])
        assert torch.equal(c, ref_c) and torch.equal(r, ref_r) and torch.equal(d, ref_d), (mode, P)
        if mode == "sparse":
            ws = max(rk.total_bytes + rk.local_bytes for rk in rast.sparse_pool.all)
        else:
            ws = _geometry_bytes(_lib.load(), rast.plan.P_pad)
        del c, r, d
        rast.close()
        with pytest.raises(RuntimeError):
            rast(means3D=t["means3D"], means2D=torch.zeros_like(t["means3D"]), opacities=t["opacities"],
                 shs=t["shs"], scales=t["scales"], rotations=t["rotations"])
        rast.close()      # a second close does nothing
        return ws

    def free():
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return torch.cuda.mem_get_info(dev)[0]

    ws = max(cycle(P) for P in sizes)   # warm-up: NCCL communicator, modules, pinned words
    start = free()
    for _ in range(5):
        for P in sizes:
            ws = max(ws, cycle(P))
    end = free()
    assert start - end <= ws, (mode, start - end, ws)


def _restated_loop(steps, P, interval, seed, max_densify_percent=0.01, min_opacity=0.005):
    """run_sharded_edit_loop at world 1, restated on one GPU: GaussianRasterizer(deterministic=True) through render()
    and the densify on the whole cloud with optim_surgery (top-k by (value desc, index asc), clones with zero moments)."""
    from types import SimpleNamespace
    from gaussianeditor_b200 import gaussian_renderer as GR, synth
    from gaussianeditor_b200.edit_loop import EditScene, make_view
    dev = torch.device("cuda", 0)
    cloud, cams = synth.make_config("c5", P=P)
    scene = EditScene(cloud, dev)
    views = [make_view(c, dev) for c in cams]
    pipe = SimpleNamespace(convert_SHs_python=False, compute_cov3D_python=False, debug=False)
    bg = torch.zeros(3, device=dev)
    with torch.no_grad():
        g = torch.Generator(device=dev).manual_seed(seed)
        targets = []
        for v in views:
            img = GR.render(v, scene, pipe, bg)["render"]
            targets.append((img + 0.05 * torch.randn(img.shape, generator=g, device=dev)).clamp(0, 1))
    rng = np.random.default_rng(seed)
    counts, losses = [], []
    attrs = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
             "scaling": "_scaling", "rotation": "_rotation"}
    for step in range(1, steps + 1):
        k = int(rng.integers(len(views)))
        pkg = GR.render(views[k], scene, pipe, bg, deterministic=True)
        sem = GR.render(views[k], scene, pipe, bg, override_color=scene.mask[..., None].float().repeat(1, 3),
                        deterministic=True)["render"]
        semantic = torch.norm(sem, dim=0) > 0.8
        loss = 10.0 * (pkg["render"] - targets[k]).abs().mean() + 0.0 * semantic.float().mean()
        scene.optimizer.zero_grad(set_to_none=True)
        loss.backward()
        with torch.no_grad():
            vis = pkg["visibility_filter"]
            scene.max_radii2D[vis] = torch.max(scene.max_radii2D[vis], pkg["radii"][vis].float())
            scene.add_densification_stats(pkg["viewspace_points"].grad, vis)
        scene.optimizer.step()
        losses.append(float(loss.detach()))
        if step % interval == 0 and step < steps:
            with torch.no_grad():
                grads = (scene.xyz_gradient_accum / scene.denom).squeeze(1)
                n = grads.numel()
                sel = SR.top_k_mask(grads, max(1, int(n * max_densify_percent)))
                keep = (torch.sigmoid(scene._opacity).squeeze(1) >= min_opacity) | sel
                kept = optim_surgery.prune_optimizer(scene.optimizer, keep)
                optim_surgery.cat_tensors_to_optimizer(scene.optimizer,
                                                       {nm: p.detach()[sel[keep]] for nm, p in kept.items()})
                scene.mask = torch.cat((scene.mask[keep], scene.mask[sel]))
                for grp in scene.optimizer.param_groups:
                    setattr(scene, attrs[grp["name"]], grp["params"][0])
                m = scene._xyz.shape[0]
                scene.max_radii2D = torch.zeros(m, device=dev)
                scene.xyz_gradient_accum = torch.zeros(m, 1, device=dev)
                scene.denom = torch.zeros(m, 1, device=dev)
        counts.append(scene._xyz.shape[0])
    params = {nm: getattr(scene, a).detach() for nm, a in attrs.items()}
    return counts, losses, params, scene


@pytest.mark.gpu
def test_sharded_edit_loop_world1_equals_single_gpu_restatement(nccl_world1):
    from gaussianeditor_b200.edit_loop import run_sharded_edit_loop
    steps, P, interval = 200, 60000, 50
    counts, losses, params, scene = _restated_loop(steps, P, interval, seed=0)
    assert len(set(counts)) > 1   # the cloud really changed size
    for mode in ("dense", "sparse"):
        out = run_sharded_edit_loop(steps=steps, P=P, densification_interval=interval, seed=0, mode=mode,
                                    deterministic=True)
        assert out["mode"] == mode and out["world"] == 1 and len(out["densify"]) == 3
        assert out["counts"] == counts, mode
        assert out["losses"] == losses, mode
        for nm, p in params.items():
            assert torch.equal(out["params"][nm], p), (mode, nm)
        assert torch.equal(out["mask"], scene.mask)
        for g, fg in zip(out["optimizer"].param_groups, scene.optimizer.param_groups):
            st, fst = out["optimizer"].state[g["params"][0]], scene.optimizer.state[fg["params"][0]]
            for key in ("exp_avg", "exp_avg_sq", "step"):
                assert torch.equal(st[key], fst[key]), (mode, g["name"], key)


# ---------------------------------------------------------------------------------------------------------------
# GPU: two processes
# ---------------------------------------------------------------------------------------------------------------
def _two_gpu_worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["LOCAL_WORLD_SIZE"] = str(world)
    res = {}
    try:
        dev = torch.device("cuda", rank)
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
        res.update(_two_gpu_body(rank, world, dev))
    except Exception:
        res["error"] = traceback.format_exc()
    finally:
        out[rank] = res
        if dist.is_initialized():
            dist.destroy_process_group()


def _gather(ex, plan, t):
    """The whole cloud's rows of a per-Gaussian tensor [plan.count, ...] (every rank gets all of them)."""
    L = plan.slice_len
    total = torch.zeros((ex.world * L,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    total[plan.rank * L:plan.rank * L + plan.count] = t
    ex.all_gather_inplace(total)
    return torch.cat([total[r * L:r * L + S.ShardPlan(plan.P_total, ex.world, r).count] for r in range(ex.world)])


def _two_gpu_body(rank, world, dev):
    from gaussianeditor_b200 import synth
    from gaussianeditor_b200.edit_loop import _SCENE_ATTR, EditScene, make_view, sharded_densify, sharded_scene
    from gaussianeditor_b200.gaussian_renderer import _settings_for
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    ex = S.Exchange()
    cloud, cams = synth.make_config("c5", P=50003)
    P = cloud.means3D.shape[0]
    plan = S.ShardPlan(P, world, rank)
    scene = sharded_scene(cloud, dev, plan)
    ok = {}
    for it in range(2):
        g = torch.Generator(device=dev).manual_seed(10 + it)   # the same full statistics on every rank
        accum_full = torch.rand(plan.P_total, 1, generator=g, device=dev).round(decimals=2)   # heavy ties
        denom_full = torch.randint(0, 3, (plan.P_total, 1), generator=g, device=dev).float()
        scene.xyz_gradient_accum = S.shard_slice(accum_full, plan).clone()
        scene.denom = S.shard_slice(denom_full, plan).clone()
        before = {a: _gather(ex, plan, getattr(scene, a).detach()) for a in _SCENE_ATTR.values()}
        mask_before = _gather(ex, plan, scene.mask)
        plan, _ = sharded_densify(scene, ex, plan)
        sel = SR.top_k_mask((accum_full / denom_full).squeeze(1), max(1, int(P * 0.01)))
        keep = (torch.sigmoid(before["_opacity"]).squeeze(1) >= 0.005) | sel
        for a in _SCENE_ATTR.values():
            ok[it, a] = torch.equal(_gather(ex, plan, getattr(scene, a).detach()),
                                    torch.cat((before[a][keep], before[a][sel])))
        ok[it, "mask"] = torch.equal(_gather(ex, plan, scene.mask), torch.cat((mask_before[keep], mask_before[sel])))
        P = plan.P_total
        view = make_view(cams[3], dev)
        rs = _settings_for(view, torch.zeros(3, device=dev), 1.0, scene.active_sh_degree)
        for mode in ("dense", "sparse"):
            rast = S.ShardedGaussianRasterizer(rs, P, mode=mode)
            with torch.no_grad():
                c, r, d = rast(means3D=scene.get_xyz, means2D=torch.zeros_like(scene._xyz), opacities=scene.get_opacity,
                               shs=scene.get_features, scales=scene.get_scaling, rotations=scene.get_rotation)
                full = {a: _gather(ex, plan, getattr(scene, a).detach()) for a in _SCENE_ATTR.values()}
                one = EditScene.__new__(EditScene)
                for a, v in full.items():
                    setattr(one, a, v)
                rc, rr, rd = GaussianRasterizer(rs)(
                    means3D=one.get_xyz, means2D=torch.zeros_like(one._xyz), opacities=one.get_opacity,
                    shs=one.get_features, scales=one.get_scaling, rotations=one.get_rotation)
            ok[it, mode] = (torch.equal(c, rc) and torch.equal(d, rd) and torch.equal(r, S.shard_slice(rr, plan)))
            del c, r, d
            rast.close()
    return {"ok": {str(k): bool(v) for k, v in ok.items()}}


@pytest.mark.gpu
def test_two_process_densify_matches_restatement():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = 2
    out = mp.Manager().dict()
    mp.spawn(_two_gpu_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    for r in range(world):
        assert "error" not in out[r], out[r].get("error")
        assert all(out[r]["ok"].values()), out[r]["ok"]
