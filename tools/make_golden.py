"""Generate the committed golden vectors under tests/golden/ by running the REFERENCE's own CUDA build
(oracle/_ref/libdgr_ref.so = the unmodified reference .cu files, see oracle/Makefile) on small seeded scenes.
Needs a GPU and the built oracle/_ref:   python tools/make_golden.py OUT_DIR   (writes OUT_DIR/*.npz; copy them to
tests/golden/ and commit).  The reference has no tests or fixtures of its own (SURVEY.md section 4); these files
are what pins the CPU oracle and our kernels to the reference's actual outputs when no GPU reference is at hand:
  * <case>.npz                    inputs and full reference outputs of four tiny scenes (tests/test_golden.py);
  * small_cases_reference.npz     (goes to tests/golden/parity/) for test_parity_gpu's small cases: SHA-256 digests of every forward output and a
                                  seeded sample of every gradient with its noise floor and max |value|;
  * reference_outputs.npz         (goes to tests/golden/parity/) every other reference value test_parity_gpu compares
                                  with: the tests that use test_parity_gpu._Ref are run here against the live reference
                                  (their assertions included) and what they computed from it is recorded;
  * camera_models_reference.npz   (goes to tests/golden/parity/) the same for tests/test_camera_models.py, written alone
                                  by   python tools/make_golden.py OUT_DIR camera_models
  * tile_grid_reference.npz       (goes to tests/golden/parity/) the same for tests/test_tile_grid.py, written alone by
                                  python tools/make_golden.py OUT_DIR tile_grid
  * magnitudes_reference.npz      (goes to tests/golden/parity/) the same for tests/test_magnitudes.py, written alone by
                                  python tools/make_golden.py OUT_DIR magnitudes
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch

from gaussianeditor_b200 import synth
import test_parity_gpu as T

import test_list_edges as LE

OUT = None


def case(name, cloud, cam, bg, colors_precomp=None, scale_modifier=1.0, seed=0):
    dL = np.random.default_rng(seed).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)
    ref = T._ref_run(cloud, cam, bg, dL=dL, colors_precomp=colors_precomp, scale_modifier=scale_modifier)
    ref2 = T._ref_run(cloud, cam, bg, dL=dL, colors_precomp=colors_precomp, scale_modifier=scale_modifier)
    s = ref["state"]
    g = ref["grads"]
    noise = {k: float((g[k] - ref2["grads"][k]).norm() / (g[k].norm() + 1e-30)) for k in g}
    np.savez_compressed(
        os.path.join(OUT, name + ".npz"),
        # inputs
        means3D=cloud.means3D, scales=cloud.scales, rotations=cloud.rotations, opacities=cloud.opacities,
        shs=cloud.shs, sh_degree=cloud.sh_degree, colors_precomp=np.zeros((0, 3), np.float32) if colors_precomp is None else colors_precomp,
        viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix, campos=cam.campos, tanfovx=cam.tanfovx,
        tanfovy=cam.tanfovy, H=cam.image_height, W=cam.image_width, bg=np.asarray(bg, np.float32),
        scale_modifier=scale_modifier, dL=dL,
        # reference outputs
        color=ref["color"].cpu().numpy(), depth=ref["depth"].cpu().numpy(), radii=ref["radii"].cpu().numpy(),
        R=ref["R"], final_T=s["final_T"].cpu().numpy(), n_contrib=s["n_contrib"].cpu().numpy(),
        ranges=s["ranges"].cpu().numpy(), point_list=s["point_list"].cpu().numpy(),
        tiles_touched=s["tiles_touched"].cpu().numpy(), means2D=s["means2D"].cpu().numpy(),
        conic_opacity=s["conic_opacity"].cpu().numpy(), rgb=s["rgb"].cpu().numpy(), depths=s["depths"].cpu().numpy(),
        **{k: v.cpu().numpy() for k, v in g.items()},
        noise=np.array([noise[k] for k in sorted(noise)]), noise_keys=np.array(sorted(noise)))
    print(name, "R", ref["R"], "visible", int((ref["radii"] > 0).sum()), "noise", max(noise.values()))


def parametrizations(fn):
    """Keyword arguments of every parameter set of a test (the product of its parametrize marks)."""
    combos = [{}]
    for m in [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]:
        names = [n.strip() for n in m.args[0].split(",")]
        combos = [dict(c, **dict(zip(names, v if isinstance(v, tuple) else (v,)))) for c in combos for v in m.args[1]]
    return combos


def main():
    global OUT
    OUT = sys.argv[1]
    os.makedirs(OUT, exist_ok=True)
    assert T.ref_cuda.available(), "oracle/_ref/libdgr_ref.so is not built"
    if sys.argv[2:] == ["camera_models"]:
        import test_camera_models as CM
        np.savez_compressed(os.path.join(OUT, "camera_models_reference.npz"),
                            **record((CM.test_forward_mark_visible_apply_weights_match_reference,)))
        print("golden written to", OUT)
        return
    if sys.argv[2:] == ["magnitudes"]:
        import test_magnitudes as MG
        np.savez_compressed(os.path.join(OUT, "magnitudes_reference.npz"),
                            **record((MG.test_forward_bit_exact_every_variant, MG.test_backward_against_reference,
                                      MG.test_translated_patch_matches_reference,
                                      MG.test_mark_visible_and_apply_weights_bit_exact)))
        print("golden written to", OUT)
        return
    if sys.argv[2:] == ["tile_grid"]:
        import test_tile_grid as TG
        np.savez_compressed(os.path.join(OUT, "tile_grid_reference.npz"),
                            **record((TG.test_lists_and_forward, TG.test_backward_against_truth,
                                     TG.test_wide_backward_against_reference)))
        print("golden written to", OUT)
        return
    c3, _ = synth.make_config("c3", P=400)
    case("c3_p400_deg3", c3, synth.ring_cameras(8, 4.5, 15.0, 72, 56, 61.0)[2], (0.1, 0.3, 0.6), seed=1)
    c1, _ = synth.make_config("c1", P=300)
    case("c1_p300_deg0", c1, synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 64, 48, fovy_deg=50.0), (0, 0, 0), seed=2)
    c2, _ = synth.make_config("c2", P=300)
    cp = np.random.default_rng(5).uniform(size=(300, 3)).astype(np.float32)
    case("c2_p300_colors_mod07", c2, synth.look_at_camera((0, 0, -3.5), (0, 0, 0), (0, -1, 0), 50, 35, fovy_deg=50.0),
         (1, 1, 1), colors_precomp=cp, scale_modifier=0.7, seed=3)
    hotspot_case()
    small = {}
    for name, cloud, cam, bg in T._small_cases():
        dL = T._small_case_dL(cam)
        ref = T._ref_run(cloud, cam, bg, dL=dL)
        ref2 = T._ref_run(cloud, cam, bg, dL=dL)
        for k, x in T._ref_forward_fields(ref).items():
            small[f"{name}/fwd/{k}"] = np.array(T._digest(x))
        for _, b in T.GRAD_PAIRS:
            r = ref["grads"][b].cpu().numpy().ravel()
            small[f"{name}/bwd/{b}"] = r[T._sample_index(r.size)]
            small[f"{name}/bwd/{b}/noise"] = np.float64(T.rel_l2(ref2["grads"][b].cpu().numpy().ravel(), r))
            small[f"{name}/bwd/{b}/absmax"] = np.float64(np.abs(r).max())
    np.savez_compressed(os.path.join(OUT, "small_cases_reference.npz"), **small)
    np.savez_compressed(os.path.join(OUT, "reference_outputs.npz"), **record(RECORDED))
    print("golden written to", OUT)


def hotspot_case():
    """A hot tile of 1500 sub-pixel splats plus densify_and_clone copies (tests/golden/hotspot_p1500_clones.npz)."""
    cloud, cam = synth.hotspot_cloud(P=1500, extra=50)
    case("hotspot_p1500_clones", synth.clone_rows(cloud), cam, (0.1, 0.2, 0.3), seed=4)


# the tests that use test_parity_gpu._Ref: run against the live reference (their assertions included), and what they
# computed from it is recorded
RECORDED = (T.test_precomputed_colors_and_scale_modifier, T.test_mark_visible_and_apply_weights_match_reference,
            T.test_apply_weights_channels_and_float_masks,
            T.test_alpha_output_matches_reference_accum_alpha_and_is_differentiable,
            T.test_binning_variants_match_reference_lists, T.test_edit_loop_matches_the_reference_rasterizer_step_by_step,
            T.test_sh_degrees_and_coefficient_counts, T.test_precomputed_covariance_path,
            T.test_hd_frame_partial_tile_row_and_debug_flag, T.test_full_size_configs_match_reference_cuda,
            T.test_needle_forward_bit_exact_every_variant, T.test_needle_backward_blend_weights_every_variant,
            T.test_frustum_edge_forward_and_preprocess_backward, T.test_opacity_edge_forward_and_backward,
            T.test_frame_size_edges, LE.test_forward_bit_exact_binning_and_depth_sort_variants,
            LE.test_backward_against_reference_and_fp64, LE.test_apply_weights_matches_reference)


def record(tests):
    T.RECORD = {}
    for fn in tests:
        for kw in parametrizations(fn):
            fn(**kw)
            print("recorded", fn.__name__, kw)
    return T.RECORD


if __name__ == "__main__":
    main()
