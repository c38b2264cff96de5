"""render_bwd variant 15 (csrc/render_bwd.cu: the per-splat moment reduction deferred and batched through shared
memory) against the reference, the fp64 CPU oracle, variant 14 and the sharded path.

Every test pins the variant with ``_options``, which restores the value it found.
Reference values fall back to the ones recorded under tests/golden/parity/ when the compiled reference is absent; they do
not depend on our variant.
"""
import numpy as np
import pytest
import torch

from gaussianeditor_b200 import synth, _lib
from oracle import cpu_oracle, ref_cuda
from util import run_ours, rel_l2, cloud_tensors, settings_from
from test_parity_gpu import (GRAD_PAIRS, _Ref, _grads_vs_reference_and_truth, _needle_case, _options, _ref_run,
                             _sample_index, _small_case_dL, _small_cases, _small_golden)

pytestmark = pytest.mark.gpu

BATCHED = 15


def test_small_cases_match_reference():
    """The three small cases of test_backward_matches_reference_cuda, with its bounds."""
    live = ref_cuda.available()
    gold = None if live else _small_golden()
    with _options(render_bwd_variant=BATCHED):
        for name, cloud, cam, bg in _small_cases():
            dL = _small_case_dL(cam)
            ours = run_ours(cloud, cam, bg, dL=dL)
            if live:
                ref = _ref_run(cloud, cam, bg, dL=dL)
                ref2 = _ref_run(cloud, cam, bg, dL=dL)
            for a, b in GRAD_PAIRS:
                g = ours["grads"][a].cpu().numpy().ravel()
                if live:
                    r = ref["grads"][b].cpu().numpy().ravel()
                    noise = rel_l2(ref2["grads"][b].cpu().numpy().ravel(), r)
                    rmax = np.abs(r).max()
                else:
                    g = g[_sample_index(g.size)]
                    r = gold[f"{name}/bwd/{b}"]
                    noise, rmax = float(gold[f"{name}/bwd/{b}/noise"]), float(gold[f"{name}/bwd/{b}/absmax"])
                err = rel_l2(g, r)
                assert err <= 1e-4 + 10 * noise, (name, a, err, noise)
                assert np.abs(g - r).max() <= 1e-3 * rmax + 1e-12, (name, a)


def test_needle_blend_weights_per_gaussian():
    """Each Gaussian's total blend weight on the needle scene (see test_needle_backward_blend_weights_every_variant):
    a dropped or an extra (pixel, splat) hit moves it by at least T/255."""
    cloud, cam, cp = _needle_case()
    H, W = cam.image_height, cam.image_width
    dL = np.zeros((3, H, W), np.float32)
    dL[1] = 1.0
    with _options(render_bwd_variant=BATCHED):
        ours = run_ours(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp)

    def compute():
        a = _ref_run(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp)["grads"]["dL_dcolors"]
        b = _ref_run(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=cp)["grads"]["dL_dcolors"]
        return dict(dL_dcolors=a, noise=(a - b).abs())
    ref = _Ref("needle/bwd", compute, full=("dL_dcolors", "noise"))
    got = ours["grads"]["dcolor"].cpu().numpy().astype(np.float64)
    want = np.asarray(ref.value("dL_dcolors"), np.float64).reshape(got.shape)
    noise = np.asarray(ref.value("noise"), np.float64).reshape(got.shape)
    tol = 3.0 * noise + 1e-5 * np.abs(want) + 1e-4
    assert np.all(got[:, [0, 2]] == 0.0) and (want[:, 1] > 0.0).mean() > 0.9
    assert (tol[:, 1] < 0.5 / 255).mean() >= 0.75
    over = np.abs(got - want) > tol
    assert not over.any(), (np.argwhere(over)[:8].tolist(), np.abs(got - want)[over][:8])


@pytest.mark.parametrize("scene", ["opacity_edge", "frustum_edge"])
def test_edge_scenes_match_reference_and_fp64(scene):
    """Opacity-edge (opacities at fp32(1/255), the 0.99 clamp, the T < 1e-4 stop) and frustum-edge scenes: all six
    gradients against the reference and the fp64 CPU oracle (5e-5)."""
    if scene == "opacity_edge":
        cloud, cam = synth.opacity_edge_cloud()
        bg, seed = (0.0, 0.5, 1.0), 44
    else:
        cloud, cam = synth.frustum_edge_cloud()
        bg, seed = (0.1, 0.2, 0.3), 43
    dL = np.random.default_rng(seed).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    with _options(render_bwd_variant=BATCHED):
        ours = run_ours(cloud, cam, bg, dL=dL)
    _grads_vs_reference_and_truth(f"{scene}/bwd", cloud, cam, bg, dL, ours, GRAD_PAIRS, 5e-5)


def _config3():
    cloud, cams = synth.make_config("c3")
    cam = cams[-1]
    dL = np.random.default_rng(11).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    return cloud, cam, (0.1, 0.2, 0.3), dL


def test_config3_full_size_matches_fp64_and_reference():
    """Config 3 at full size: every gradient within 5e-5 relative L2 of the fp64 CPU oracle, and against the reference
    as in test_full_size_configs_match_reference_cuda (whose recorded values this reads when the reference is absent)."""
    cloud, cam, bg, dL = _config3()
    with _options(render_bwd_variant=BATCHED):
        ours = run_ours(cloud, cam, bg, dL=dL)
    f64 = cpu_oracle.forward_from(cloud, cam, bg, f32=False)
    truth = f64.backward(dL)
    f64.close()

    def compute():
        ref = _ref_run(cloud, cam, bg, dL=dL)
        ref2 = _ref_run(cloud, cam, bg, dL=dL)
        s = ref["state"]
        out = dict(R=ref["R"], radii=ref["radii"], color=ref["color"], depth=ref["depth"],
                   n_contrib=s["n_contrib"].flatten(), final_T=s["final_T"].flatten(), point_list=s["point_list"])
        for a, b in GRAD_PAIRS:
            r = ref["grads"][b].cpu().numpy()
            out[b] = r
            out["noise/" + b] = rel_l2(ref2["grads"][b].cpu().numpy(), r)
            out["ref_err/" + b] = rel_l2(r, truth[a])
        return out
    ref = _Ref("full_size/c3", compute, close=[b for _, b in GRAD_PAIRS])
    assert ours["R"] == ref.scalar("R")
    for name, x in [("radii", ours["radii"]), ("color", ours["color"]), ("depth", ours["depth"])]:
        assert ref.equal(name, x), name
    for a, b in GRAD_PAIRS:
        g = ours["grads"][a].cpu().numpy()
        ours_err = rel_l2(g, truth[a])
        assert ours_err <= 5e-5, (a, ours_err)
        noise, ref_err = ref.scalar("noise/" + b), ref.scalar("ref_err/" + b)
        assert ref_err <= 1.5e-3, (a, ref_err)
        err = rel_l2(*ref.pair(b, g))
        assert err <= 1e-4 + 10 * noise + 1.5 * ref_err, (a, err, noise, ref_err)


def test_config3_matches_variant14():
    """The same config-3 step under variants 15 and 14: the forward is shared (bit-identical), and the gradients differ
    only in the order of the fp32 sums (5e-5 relative L2 per tensor)."""
    cloud, cam, bg, dL = _config3()
    out = {}
    for v in (BATCHED, 14):
        with _options(render_bwd_variant=v):
            out[v] = run_ours(cloud, cam, bg, dL=dL)
    a, b = out[BATCHED], out[14]
    assert a["R"] == b["R"]
    for k in ("color", "depth", "radii"):
        assert torch.equal(a[k], b[k]), k
    for name, _ in GRAD_PAIRS:
        err = rel_l2(a["grads"][name].cpu().numpy(), b["grads"][name].cpu().numpy())
        assert err <= 5e-5, (name, err)


def test_sparse_sharded_virtual_ranks_match_single_gpu():
    """Three virtual ranks of the sparse Gaussian-sharded path on one GPU (tile-row ownership in the kernel) against
    the single-GPU rasterizer, both with variant 15: frames bit-exact, gradients to summation order."""
    from gaussianeditor_b200 import sharded as S
    from gaussianeditor_b200 import sparse_sharded as SS
    dev = torch.device("cuda")
    world = 3
    cloud, cams = synth.make_config("c3", P=60013)
    cam = cams[0]
    bg = (0.2, 0.5, 0.1)
    dL = np.random.default_rng(3).random((3, cam.image_height, cam.image_width), dtype=np.float32)
    H, W = cam.image_height, cam.image_width
    with _options(render_bwd_variant=BATCHED):
        ref = run_ours(cloud, cam, bg=bg, dL=dL)
        rs = settings_from(cam, bg, cloud.sh_degree, dev)
        full = cloud_tensors(cloud, dev)
        P = cloud.means3D.shape[0]
        empty = torch.empty(0, device=dev)
        ranks = [SS.SparseRank(S.ShardPlan(P, world, r), dev, W, H) for r in range(world)]
        SS.link_virtual(ranks)
        for rk in ranks:
            rk.matrix.zero_()
        steps = []
        for rk in ranks:
            sl = lambda t: S.shard_slice(t, rk.plan)
            steps.append(SS.sparse_preprocess(rk, rs, sl(full["means3D"]), sl(full["shs"]), empty, sl(full["opacities"]),
                                              sl(full["scales"]), sl(full["rotations"]), empty, ranks[0].cap_alloc))
        matrix = torch.stack([rk.matrix for rk in ranks]).sum(0)
        for rk in ranks:
            rk.matrix.copy_(matrix)
        out = [SS.sparse_order(st) for st in steps]
        assert sum(o[0] for o in out) == ref["R"]
        for st in steps:
            SS.sparse_render(st, st.rk.frame[:3], st.rk.frame[3:])
        for rk in ranks:
            SS.frame_broadcast(rk)
        torch.cuda.synchronize()
        for rk in ranks:
            assert torch.equal(rk.frame[:3], ref["color"]) and torch.equal(rk.frame[3:], ref["depth"]), rk.plan.rank
        gdL = torch.from_numpy(dL).to(dev)
        accs = [SS.sparse_backward_render(st, gdL) for st in steps]
        for st, acc in zip(steps, accs):
            SS.sparse_return(st, acc)
        names = ["dmean3D", "dmean2D", "dsh", None, "dopacity", "dscale", "drot", None]
        for st in steps:
            p = st.rk.plan
            grads = SS.sparse_backward_preprocess(st)
            for name, g in zip(names, grads):
                if name is None:
                    continue
                want = ref["grads"][name][p.base:p.base + p.count]
                assert g.shape == want.shape
                assert rel_l2(g.cpu().numpy(), want.cpu().numpy()) <= 2e-5, (name, p.rank)
