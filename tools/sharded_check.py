"""One process per GPU (torchrun): the Gaussian-sharded rasterizer must reproduce the single-GPU rasterizer.

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/sharded_check.py [--config c2 --P N]

Every rank renders the full cloud alone (single-GPU path) and then its shard through ShardedGaussianRasterizer;
images and radii must be bit-identical, gradients within 2e-5 relative L2. Prints SHARDED_CHECK_OK on rank 0.
"""
import argparse
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from gaussianeditor_b200 import sharded as S, synth  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer  # noqa: E402
from util import cloud_tensors, rel_l2, settings_from  # noqa: E402


def check_apply_weights(rast, full, loc, cams, bg, sh_degree, dev):
    """Semantic tracing on the shard vs the full cloud: two views accumulated into the same rows (CH = 1 with a binary
    mask, CH = 3 with a float mask), `cnt` bit-identical, `weights` within the float-sum bounds, rows that no splat hits
    untouched; markVisible equals the slice of the full-cloud result. The masks are identical on every rank."""
    plan = rast.plan
    P = full["means3D"].shape[0]
    ok, worst = True, 0.0
    m3, op = full["means3D"].detach(), full["opacities"].detach()
    sc, ro = full["scales"].detach(), full["rotations"].detach()
    lm3, lop, lsc, lro = (loc[k].detach() for k in ("means3D", "opacities", "scales", "rotations"))
    for CH, binary in ((1, True), (3, False)):
        w_ref = torch.zeros(P, CH, device=dev); c_ref = torch.zeros(P, 1, dtype=torch.int32, device=dev)
        w = torch.full((plan.count, CH), 7.0, device=dev); c = torch.full((plan.count, 1), 5, dtype=torch.int32, device=dev)
        for i, cam in enumerate(cams[:2]):
            rs = settings_from(cam, bg, sh_degree, dev)
            g = torch.Generator().manual_seed(100 * CH + i)
            m = torch.rand(CH, cam.image_height, cam.image_width, generator=g)
            iw = ((m > 0.5).float() if binary else m).to(dev)
            GaussianRasterizer(rs).apply_weights(m3, None, op, None, w_ref, sc, ro, None, c_ref, iw)
            rast.raster_settings = rs
            rast.apply_weights(lm3, None, lop, None, w, lsc, lro, None, c, iw)
            if i == 0:
                vis = rast.markVisible(lm3)
                ok = ok and torch.equal(vis, S.shard_slice(GaussianRasterizer(rs).markVisible(m3), plan))
        wr, cr = S.shard_slice(w_ref, plan), S.shard_slice(c_ref, plan)
        ok = ok and torch.equal(c - 5, cr) and bool((w[(cr == 0).view(-1)] == 7.0).all())
        dw = w - 7.0
        if binary:
            ok = ok and torch.equal(dw, wr)
        else:
            worst = max(worst, rel_l2(dw.cpu().numpy(), wr.cpu().numpy()))
            ok = ok and float((dw - wr).abs().max()) <= 1e-4 * float(wr.abs().max())
    ok = ok and worst <= 1e-5
    return ok, f" apply_weights_worst_rel_l2={worst:.2e}"


def check_deterministic(a, cloud, cams, bg, dL, dev, rank, world):
    """ShardedGaussianRasterizer(deterministic=True) under torch's deterministic flag: two identical fwd+bwd steps and
    two identical traces (two views, CH = 1 binary and CH = 3 float masks) must give the same bits; at world 1 they must
    also equal GaussianRasterizer(deterministic=True). Returns (ok, digest of every rank's results, message)."""
    import hashlib
    P = cloud.means3D.shape[0]
    rs = settings_from(cams[0], bg, cloud.sh_degree, dev)
    view_rs = [settings_from(cam, bg, cloud.sh_degree, dev) for cam in cams[:2]]
    torch.use_deterministic_algorithms(True)
    if a.no_fill:
        from torch.utils import deterministic as torch_det
        torch_det.fill_uninitialized_memory = False
    rast = S.ShardedGaussianRasterizer(rs, P, p2p=(True if a.mode == 'sparse' else a.p2p), mode=a.mode,
                                       deterministic=True)
    plan = rast.plan
    full = cloud_tensors(cloud, dev)

    def step(r, tensors):
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in tensors.items()}
        m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
        color, _, _ = r(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], shs=leaves["shs"],
                        scales=leaves["scales"], rotations=leaves["rotations"])
        (color * dL).sum().backward()
        out = {k: v.grad for k, v in leaves.items()}
        out["means2D"] = m2.grad
        for CH, binary in ((1, True), (3, False)):
            n = tensors["means3D"].shape[0]
            w = torch.zeros(n, CH, device=dev); c = torch.zeros(n, 1, dtype=torch.int32, device=dev)
            for i, cam in enumerate(cams[:2]):
                r.raster_settings = view_rs[i]
                g = torch.Generator().manual_seed(100 * CH + i)
                m = torch.rand(CH, cam.image_height, cam.image_width, generator=g)
                iw = ((m > 0.5).float() if binary else m).to(dev)
                r.apply_weights(tensors["means3D"], None, tensors["opacities"], None, w, tensors["scales"],
                                tensors["rotations"], None, c, iw)
            r.raster_settings = rs
            out[f"weights{CH}"], out[f"cnt{CH}"] = w, c
        torch.cuda.synchronize()
        return {k: v.detach().cpu().clone() for k, v in out.items()}

    loc = {k: S.shard_slice(v, plan) for k, v in full.items()}
    runs = [step(rast, loc) for _ in range(2)]
    bits = lambda d: {k: v.numpy().tobytes() for k, v in d.items()}
    ok = bits(runs[0]) == bits(runs[1])
    if world == 1:
        ref = step(GaussianRasterizer(rs, deterministic=True), full)
        ok = ok and all(torch.equal(runs[0][k], ref[k]) for k in ref)
    mine = hashlib.sha256(b"".join(v for _, v in sorted(bits(runs[0]).items()))).hexdigest()
    digests = [None] * world
    dist.all_gather_object(digests, mine)
    rast.close()
    torch.use_deterministic_algorithms(False)
    return ok, hashlib.sha256("".join(digests).encode()).hexdigest(), " deterministic=" + ("ok" if ok else "FAILED")


def raw_params(t):
    """The scene model's raw parameters of a cloud (the inverse activations; rotations left unnormalised)."""
    o = t["opacities"].clamp(1e-6, 1 - 1e-6)
    return dict(means3D=t["means3D"], opacity_logits=torch.log(o / (1 - o)), features_dc=t["shs"][:, :1].contiguous(),
                features_rest=t["shs"][:, 1:].contiguous(), log_scales=torch.log(t["scales"]),
                raw_rotations=t["rotations"] * 1.7)


def check_fused_depth(a, cloud, cam, bg, dL, dev):
    """--raw (forward_raw on the local rows) and/or --depth-grad (depth_grad=True with a colour + depth loss, then a
    depth-only loss) against GaussianRasterizer with the same options on the full cloud: frames and radii bit-identical,
    every gradient (means2D included) within 2e-5 relative L2."""
    P = cloud.means3D.shape[0]
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    dD = torch.from_numpy(np.random.default_rng(5).random((1, cam.image_height, cam.image_width),
                                                          dtype=np.float32)).to(dev)
    t = cloud_tensors(cloud, dev)
    params = raw_params(t) if a.raw else dict(means3D=t["means3D"], opacities=t["opacities"], shs=t["shs"],
                                              scales=t["scales"], rotations=t["rotations"])
    rast = S.ShardedGaussianRasterizer(rs, P, p2p=(True if a.mode == 'sparse' else a.p2p), mode=a.mode,
                                       depth_grad=a.depth_grad)
    ref_rast = GaussianRasterizer(rs, depth_grad=a.depth_grad)

    def run(r, tensors, loss):
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in tensors.items()}
        m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
        if a.raw:
            color, radii, depth = r.forward_raw(leaves["means3D"], m2, leaves["opacity_logits"], leaves["features_dc"],
                                                leaves["features_rest"], leaves["log_scales"], leaves["raw_rotations"])
        else:
            color, radii, depth = r(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"],
                                    shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"])
        {"color": (color * dL).sum(), "both": (color * dL).sum() + (depth * dD).sum(),
         "depth": (depth * dD).sum()}[loss].backward()
        grads = {k: v.grad for k, v in leaves.items()}
        grads["means2D"] = m2.grad
        return color.detach(), radii, depth.detach(), grads

    ok, worst = True, 0.0
    for loss in (("both", "depth") if a.depth_grad else ("color",)):
        ref = run(ref_rast, params, loss)
        mine = run(rast, {k: S.shard_slice(v, rast.plan) for k, v in params.items()}, loss)
        torch.cuda.synchronize()
        ok = ok and torch.equal(mine[0], ref[0]) and torch.equal(mine[2], ref[2])
        ok = ok and torch.equal(mine[1], S.shard_slice(ref[1], rast.plan))
        for k, g in mine[3].items():
            worst = max(worst, rel_l2(g.cpu().numpy(), S.shard_slice(ref[3][k], rast.plan).cpu().numpy()))
    rast.close()
    ok = ok and worst <= 2e-5
    return ok, f" raw={a.raw} depth_grad={a.depth_grad} fused_depth_worst_rel_l2={worst:.2e}" + \
        (" fused_depth=ok" if ok else " fused_depth=FAILED")


def check_alpha_camera(a, cloud, cam, bg, dL, dev, world):
    """--alpha and/or --camera-grad (with depth_grad=True) against GaussianRasterizer with the same options on the full
    cloud, for a colour + alpha + depth loss (the alpha term only with --alpha): colour, depth, alpha and radii
    bit-identical; per-Gaussian gradients within 2e-5 relative L2; each camera array within 1e-4 relative L2 (or 10x
    the single-GPU call-to-call spread if larger) and the same bits on every rank."""
    import hashlib
    P = cloud.means3D.shape[0]
    base = settings_from(cam, bg, cloud.sh_degree, dev)
    g = np.random.default_rng(11)
    dD = torch.from_numpy(g.random((1, cam.image_height, cam.image_width), dtype=np.float32) * 0.1).to(dev)
    dA = torch.from_numpy(g.random((1, cam.image_height, cam.image_width), dtype=np.float32) - 0.5).to(dev)
    t = cloud_tensors(cloud, dev)
    cam_keys = ("viewmatrix", "projmatrix", "campos")
    opts = dict(return_alpha=a.alpha, camera_grad=a.camera_grad, depth_grad=True)

    def settings():
        if not a.camera_grad:
            return base
        return base._replace(**{k: getattr(base, k).clone().requires_grad_(True) for k in cam_keys})

    def run(make, tensors):
        rs = settings()
        r = make(rs)
        leaves = {k: v.detach().clone().requires_grad_(True) for k, v in tensors.items()}
        m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
        out = r(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], shs=leaves["shs"],
                scales=leaves["scales"], rotations=leaves["rotations"])
        loss = (out[0] * dL).sum() + (out[2] * dD).sum() + ((out[3] * dA).sum() if a.alpha else 0.0)
        loss.backward()
        grads = {k: v.grad for k, v in leaves.items()}
        grads["means2D"] = m2.grad
        cams = {k: getattr(rs, k).grad for k in cam_keys} if a.camera_grad else {}
        torch.cuda.synchronize()
        return [o.detach() for o in out], grads, cams

    rast = S.ShardedGaussianRasterizer(base, P, p2p=(True if a.mode == 'sparse' else a.p2p), mode=a.mode, **opts)
    ref_out, ref_g, ref_c = run(lambda rs: GaussianRasterizer(rs, **opts), t)
    _, _, ref_c2 = run(lambda rs: GaussianRasterizer(rs, **opts), t)
    out, grads, cams = run(lambda rs: (setattr(rast, "raster_settings", rs), rast)[1],
                           {k: S.shard_slice(v, rast.plan) for k, v in t.items()})
    ok = all(torch.equal(out[i], ref_out[i]) for i in (0, 2) + ((3,) if a.alpha else ()))
    ok = ok and torch.equal(out[1], S.shard_slice(ref_out[1], rast.plan))
    worst = max(rel_l2(v.cpu().numpy(), S.shard_slice(ref_g[k], rast.plan).cpu().numpy()) for k, v in grads.items())
    ok = ok and worst <= 2e-5
    cworst, spread = 0.0, 0.0
    for k in cams:
        spread = max(spread, rel_l2(ref_c2[k].cpu().numpy(), ref_c[k].cpu().numpy()))
        cworst = max(cworst, rel_l2(cams[k].cpu().numpy(), ref_c[k].cpu().numpy()))
    ok = ok and cworst <= max(1e-4, 10 * spread)
    if a.camera_grad:
        ok = ok and not cams["viewmatrix"][:, 3].any() and not cams["projmatrix"][:, 2].any()
        mine = hashlib.sha256(b"".join(cams[k].cpu().numpy().tobytes() for k in cam_keys)).hexdigest()
        digests = [None] * world
        dist.all_gather_object(digests, mine)
        ok = ok and len(set(digests)) == 1
    rast.close()
    return ok, (f" alpha={a.alpha} camera_grad={a.camera_grad} alpha_camera_worst_rel_l2={worst:.2e}"
                f" camera_worst_rel_l2={cworst:.2e} camera_spread={spread:.2e}") + \
        (" alpha_camera=ok" if ok else " alpha_camera=FAILED")


def check_static(a, cloud, cams, bg, dL, dev, world):
    """--static: ShardedGaussianRasterizer(static_capacity=N) with deterministic, alpha and depth (and, in a second run,
    camera) gradients. Per camera, the eager static step must equal the default step bit for bit (frames, radii,
    gradients, camera gradients) with status[1] == 0; a forward + backward captured in a CUDA graph and replayed for the
    cameras must equal the eager static calls bit for bit, status included; and in sparse mode the control blocks'
    epoch counters must advance by (device barriers per step) x (replays)."""
    from gaussianeditor_b200.rasterizer import _RasterizeGaussians
    P = cloud.means3D.shape[0]
    t = cloud_tensors(cloud, dev)
    views = cams[:3]
    g = np.random.default_rng(11)
    H, W = views[0].image_height, views[0].image_width
    dD = torch.from_numpy(g.random((1, H, W), dtype=np.float32) * 0.1).to(dev)
    dA = torch.from_numpy(g.random((1, H, W), dtype=np.float32) - 0.5).to(dev)
    cam_keys = ("viewmatrix", "projmatrix", "campos")
    R_max = 0
    for v in views:   # N = 1.25 x the largest R + 4096 (the single-GPU R bounds every rank's)
        GaussianRasterizer(settings_from(v, bg, cloud.sh_degree, dev))(
            means3D=t["means3D"], means2D=torch.zeros_like(t["means3D"]), opacities=t["opacities"], shs=t["shs"],
            scales=t["scales"], rotations=t["rotations"])
        R_max = max(R_max, int(_RasterizeGaussians.last_state.num_rendered))
    N = int(1.25 * R_max) + 4096
    ok, msg = True, ""
    for camera in (False, True):
        opts = dict(deterministic=True, return_alpha=True, depth_grad=True, camera_grad=camera)
        p2p = True if a.mode == "sparse" else a.p2p
        base = settings_from(views[0], bg, cloud.sh_degree, dev)
        srs = base._replace(**{k: getattr(base, k).clone().requires_grad_(camera) for k in cam_keys})
        default = S.ShardedGaussianRasterizer(base, P, p2p=p2p, mode=a.mode, **opts)
        static = S.ShardedGaussianRasterizer(srs, P, p2p=p2p, mode=a.mode, static_capacity=N, **opts)
        plan = static.plan
        leaves = {k: S.shard_slice(v, plan).clone().requires_grad_(True) for k, v in t.items()}
        m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)

        def step(r):
            out = r(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], shs=leaves["shs"],
                    scales=leaves["scales"], rotations=leaves["rotations"])
            ((out[0] * dL).sum() + (out[2] * dD).sum() + (out[3] * dA).sum()).backward()
            return out

        def clear():
            for v in list(leaves.values()) + [m2] + ([getattr(srs, k) for k in cam_keys] if camera else []):
                v.grad = None

        def result(out, rs):
            grads = [v.grad.clone() for v in list(leaves.values()) + [m2]]
            cgrads = [getattr(rs, k).grad.clone() for k in cam_keys] if camera else []
            return [o.detach().clone() for o in out], grads, cgrads

        def set_view(v):
            rs = settings_from(v, bg, cloud.sh_degree, dev)
            with torch.no_grad():
                for k in cam_keys:
                    getattr(srs, k).copy_(getattr(rs, k))
            return rs

        def same(x, y):
            return all(torch.equal(p, q) for p, q in zip(x[0] + x[1] + x[2], y[0] + y[1] + y[2]))

        eager, stat = [], []
        for v in views:
            rs = settings_from(v, bg, cloud.sh_degree, dev)
            if camera:
                rs = rs._replace(**{k: getattr(rs, k).clone().requires_grad_(True) for k in cam_keys})
            default.raster_settings = rs
            clear()
            ref = result(step(default), rs)
            set_view(v)
            clear()
            got = result(step(static), srs)
            stat.append((got, static.status.clone()))
            ok = ok and same(ref, got) and int(static.status[1]) == 0 and static.check_capacity() >= 0
            eager.append(ref)
        # capture one forward + backward after an eager warm-up on a side stream, then replay it for every view
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                clear()
                step(static)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        clear()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = step(static)
        epochs = lambda: sum(int(rk.epoch_word[0]) for rk in static.sparse_pool.all) if a.mode == "sparse" else 0
        e0 = epochs()
        for v, (want, want_status) in zip(views, stat):
            set_view(v)
            graph.replay()
            torch.cuda.synchronize()
            got = ([o.detach() for o in out], [v.grad for v in list(leaves.values()) + [m2]],
                   [getattr(srs, k).grad for k in cam_keys] if camera else [])
            ok = ok and same(want, got) and torch.equal(static.status, want_status)
        per_step = (3 + (1 if camera else 0)) if a.mode == "sparse" else 0   # row, frame, return (+ camera) barriers
        ok = ok and epochs() - e0 == per_step * len(views)
        msg += f" static(camera={camera}) N={N} epochs+={epochs() - e0}"
        del out, graph
        import gc
        gc.collect()
        torch.cuda.synchronize()
        default.close()
        static.close()
    return ok, msg + (" static=ok" if ok else " static=FAILED")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c3")
    ap.add_argument("--P", type=int, default=None)
    ap.add_argument("--p2p", action="store_true", help="dense mode: fused preprocess + all-gather over peer memory")
    ap.add_argument("--mode", default="dense", choices=["dense", "sparse"])
    ap.add_argument("--apply-weights", action="store_true",
                    help="also check semantic tracing (CH = 1 and 3) and markVisible against the full cloud")
    ap.add_argument("--deterministic", action="store_true",
                    help="also check deterministic=True under torch's deterministic flag (repeatable bits; at world 1 "
                         "the single-GPU deterministic bits); prints DETERMINISTIC_DIGEST")
    ap.add_argument("--raw", action="store_true",
                    help="also check forward_raw (fused activations) on the local rows against the single-GPU one")
    ap.add_argument("--depth-grad", action="store_true",
                    help="also check depth_grad=True with a colour + depth loss and a depth-only loss")
    ap.add_argument("--alpha", action="store_true",
                    help="also check return_alpha=True (alpha frame and a loss on it) against the single-GPU one")
    ap.add_argument("--camera-grad", action="store_true",
                    help="also check camera_grad=True: camera gradients of the whole cloud, the same bits on every rank")
    ap.add_argument("--no-fill", action="store_true",
                    help="with --deterministic: torch.utils.deterministic.fill_uninitialized_memory = False")
    ap.add_argument("--static", action="store_true",
                    help="check only static_capacity: eager static == default, captured + replayed == eager")
    a = ap.parse_args()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    S.init_distributed("nccl", dev)
    cloud, cams = synth.make_config(a.config, P=a.P)
    if a.static:
        st_ok, st_msg = check_static(a, cloud, cams, (0.2, 0.5, 0.1), torch.from_numpy(np.random.default_rng(3).random(
            (3, cams[0].image_height, cams[0].image_width), dtype=np.float32)).to(dev), dev, world)
        flag = torch.tensor([1 if st_ok else 0], device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if rank == 0:
            print(f"world={world} mode={a.mode} p2p={a.p2p}{st_msg}")
            print("SHARDED_CHECK_OK" if int(flag) == 1 else "SHARDED_CHECK_FAILED")
        dist.destroy_process_group()
        sys.exit(0 if int(flag) == 1 else 1)
    cam = cams[0]
    bg = (0.2, 0.5, 0.1)
    H, W = cam.image_height, cam.image_width
    P = cloud.means3D.shape[0]
    rs = settings_from(cam, bg, cloud.sh_degree, dev)
    dL = torch.from_numpy(np.random.default_rng(3).random((3, H, W), dtype=np.float32)).to(dev)

    full = cloud_tensors(cloud, dev, requires_grad=True)
    m2 = torch.zeros_like(full["means3D"], requires_grad=True)
    color, radii, depth = GaussianRasterizer(rs)(means3D=full["means3D"], means2D=m2, opacities=full["opacities"],
                                                shs=full["shs"], scales=full["scales"], rotations=full["rotations"])
    (color * dL).sum().backward()

    rast = S.ShardedGaussianRasterizer(rs, P, p2p=(True if a.mode == 'sparse' else a.p2p), mode=a.mode)
    plan = rast.plan
    loc = {k: S.shard_slice(v.detach(), plan).clone().requires_grad_(True) for k, v in full.items()}
    lm2 = torch.zeros_like(loc["means3D"], requires_grad=True)
    scolor, sradii, sdepth = rast(means3D=loc["means3D"], means2D=lm2, opacities=loc["opacities"], shs=loc["shs"],
                                  scales=loc["scales"], rotations=loc["rotations"])
    (scolor * dL).sum().backward()
    torch.cuda.synchronize()

    # GaussianEditor's step shape: two forwards alive at once (SH render + mask render with precomputed colours), then
    # ONE backward through the first -- exercises the workspace pool with two workspaces in flight
    torch.manual_seed(7)
    mask_col = torch.rand(plan.count, 3, device=dev)
    full_col = torch.zeros(P, 3, device=dev)
    full_col[plan.base:plan.base + plan.count] = mask_col
    dist.all_reduce(full_col)
    for v in list(loc.values()) + [lm2]:
        v.grad = None
    c1, _, _ = rast(means3D=loc["means3D"], means2D=lm2, opacities=loc["opacities"], shs=loc["shs"],
                    scales=loc["scales"], rotations=loc["rotations"])
    c2, _, _ = rast(means3D=loc["means3D"].detach(), means2D=torch.zeros_like(lm2), opacities=loc["opacities"].detach(),
                    colors_precomp=mask_col, scales=loc["scales"].detach(), rotations=loc["rotations"].detach())
    (c1 * dL).sum().backward()
    ref_c2, _, _ = GaussianRasterizer(rs)(means3D=full["means3D"].detach(), means2D=torch.zeros_like(m2),
                                          opacities=full["opacities"].detach(), colors_precomp=full_col,
                                          scales=full["scales"].detach(), rotations=full["rotations"].detach())
    two_ok = torch.equal(c1, color) and torch.equal(c2, ref_c2)
    del c1, c2
    if a.p2p or a.mode == 'sparse':  # second round through the recycled peer workspace
        for v in list(loc.values()) + [lm2]:
            v.grad = None
        del scolor, sradii, sdepth
        scolor, sradii, sdepth = rast(means3D=loc["means3D"], means2D=lm2, opacities=loc["opacities"], shs=loc["shs"],
                                      scales=loc["scales"], rotations=loc["rotations"])
        (scolor * dL).sum().backward()
        torch.cuda.synchronize()
    ok = two_ok and torch.equal(scolor, color) and torch.equal(sdepth, depth) and torch.equal(sradii, S.shard_slice(radii, plan))
    worst = 0.0
    pairs = [(loc[k].grad, S.shard_slice(full[k].grad, plan)) for k in loc] + [(lm2.grad, S.shard_slice(m2.grad, plan))]
    for g, w in pairs:
        worst = max(worst, rel_l2(g.cpu().numpy(), w.cpu().numpy()))
    ok = ok and worst <= 2e-5
    aw_msg = ""
    if a.apply_weights:
        aw_ok, aw_msg = check_apply_weights(rast, full, loc, cams, bg, cloud.sh_degree, dev)
        ok = ok and aw_ok
    if a.raw or a.depth_grad:
        fd_ok, fd_msg = check_fused_depth(a, cloud, cam, bg, dL, dev)
        ok = ok and fd_ok
        aw_msg += fd_msg
    if a.alpha or a.camera_grad:
        ac_ok, ac_msg = check_alpha_camera(a, cloud, cam, bg, dL, dev, world)
        ok = ok and ac_ok
        aw_msg += ac_msg
    det_digest = None
    if a.deterministic:
        det_ok, det_digest, det_msg = check_deterministic(a, cloud, cams, bg, dL, dev, rank, world)
        ok = ok and det_ok
        aw_msg += det_msg
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        extra = ""
        if a.mode == "sparse":
            from gaussianeditor_b200 import sparse_sharded as SS
            extra = f" sparse={SS._SparseShardedRasterize.last} redo={rast.sparse_pool.redo}"
        else:
            extra = f" R_rank0={S._ShardedRasterize.last_R}"
        print(f"world={world} mode={a.mode} p2p={a.p2p} P={P}{extra} worst_grad_rel_l2={worst:.2e}{aw_msg}")
        if det_digest is not None:
            print(f"DETERMINISTIC_DIGEST {det_digest}")
        print("SHARDED_CHECK_OK" if int(flag) == 1 else "SHARDED_CHECK_FAILED")
    del scolor, sradii, sdepth
    import gc
    gc.collect()
    rast.close()
    dist.destroy_process_group()
    sys.exit(0 if int(flag) == 1 else 1)


if __name__ == "__main__":
    main()
