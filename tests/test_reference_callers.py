"""The reference's OWN callers of the hot path, recorded by tools/make_caller_golden.py into
tests/golden/callers/reference_callers.npz (the reference's modules imported unchanged, with ``diff_gaussian_rasterization``
resolving to THIS repository's drop-in package and ``plyfile`` / ``simple_knn`` stubbed):

  * gaussiansplatting/gaussian_renderer/__init__.py and scene/gaussian_model.py: every name, keyword and positional
    slot the reference uses on the rasterizer must exist here (SURVEY 7.3-10 / 8(f-2));
  * the reference's optimizer surgery (scene/gaussian_model.py:553-641) run on CPU tensors: parameters, returned
    tensors and Adam state of gaussianeditor_b200/optim_surgery.py must equal the recorded ones bit for bit. Inputs and
    Adam state come from numpy's seeded generator and the surgery only moves data, so the recorded bits do not depend
    on the CPU's vector unit; the one Adam step afterwards is compared in-process against an Adam rebuilt from the
    reference's recorded state;
  * the reference's ``save_ply`` (:410-445): the structured array it hands to plyfile (field names, order, float32
    values) must serialise to exactly the bytes gaussianeditor_b200/ply_io.py writes behind the header, and our reader
    must give back every recorded column.
"""
import inspect
import json
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "callers", "reference_callers.npz")
GROUPS = [("xyz", 1.6e-4), ("f_dc", 2.5e-3), ("f_rest", 1.25e-4), ("opacity", 0.05), ("scaling", 5e-3), ("rotation", 1e-3)]
PLY_DEGREES = [0, 1, 3]


@pytest.fixture(scope="module")
def gold():
    z = np.load(GOLDEN)
    return z, json.loads(str(z["api"]))


def _normal(rng, *shape):
    return torch.from_numpy(rng.standard_normal(shape).astype(np.float32))


def bare_model(P=13, deg=2, seed=0):
    """Parameters and non-trivial Adam state (step 3, seeded moments) of a GaussianModel, from numpy's seeded generator."""
    rng = np.random.default_rng(seed)
    K = (deg + 1) ** 2 - 1
    shapes = {"xyz": (P, 3), "f_dc": (P, 1, 3), "f_rest": (P, K, 3), "opacity": (P, 1), "scaling": (P, 3),
              "rotation": (P, 4)}
    params = {n: torch.nn.Parameter(_normal(rng, *shapes[n])) for n, _ in GROUPS}
    opt = torch.optim.Adam([{"params": [params[n]], "lr": lr, "name": n} for n, lr in GROUPS], lr=0.0, eps=1e-15)
    for n, _ in GROUPS:
        opt.state[params[n]] = {"step": torch.tensor(3.0), "exp_avg": _normal(rng, *shapes[n]),
                                "exp_avg_sq": _normal(rng, *shapes[n]).abs()}
    return params, opt


def surgery_inputs():
    """Mask, extension tensors and replacement opacity of the surgery test (numpy's seeded generator)."""
    rng = np.random.default_rng(5)
    keep = torch.from_numpy(rng.uniform(size=13) > 0.4)
    ext = {"xyz": _normal(rng, 4, 3), "f_dc": _normal(rng, 4, 1, 3), "f_rest": _normal(rng, 4, 8, 3),
           "opacity": _normal(rng, 4, 1), "scaling": _normal(rng, 4, 3), "rotation": _normal(rng, 4, 4)}
    return rng, keep, ext


def adam_from(z, tag):
    """An Adam over fresh parameters holding the state recorded under `tag` (the reference's, after its surgery)."""
    params = {n: torch.nn.Parameter(torch.from_numpy(z[f"{tag}/{n}/param"].copy())) for n, _ in GROUPS}
    opt = torch.optim.Adam([{"params": [params[n]], "lr": lr, "name": n} for n, lr in GROUPS], lr=0.0, eps=1e-15)
    for n, _ in GROUPS:
        opt.state[params[n]] = {k: torch.from_numpy(z[f"{tag}/{n}/{k}"].copy()) for k in ("step", "exp_avg", "exp_avg_sq")}
    return opt


def adam_step(opt):
    opt.zero_grad()
    sum((gr["params"][0] ** 2).sum() for gr in opt.param_groups).backward()
    opt.step()


def snapshot(opt, tag):
    """{tag/group/param|exp_avg|exp_avg_sq|step: array} of an optimizer."""
    out = {}
    for gr in opt.param_groups:
        p = gr["params"][0]
        out[f"{tag}/{gr['name']}/param"] = p.detach().numpy().copy()
        for k, v in opt.state.get(p, {}).items():
            out[f"{tag}/{gr['name']}/{k}"] = (v.numpy() if torch.is_tensor(v) else np.asarray(v)).copy()
    return out


def returned(d, tag):
    return {f"{tag}/ret/{k}": v.detach().numpy().copy() for k, v in d.items()}


def _assert_recorded(z, got, tag):
    want = sorted(k for k in z.files if k.startswith(tag + "/"))
    assert sorted(got) == want, tag
    for k in want:
        assert got[k].dtype == z[k].dtype and np.array_equal(got[k], z[k]), k


def test_reference_render_uses_only_names_the_drop_in_has(gold):
    import diff_gaussian_rasterization as dgr
    import gaussianeditor_b200.rasterizer as RZ
    _, api = gold
    # the reference's renderer imports these names from diff_gaussian_rasterization: they are the drop-in's classes
    assert {"GaussianRasterizer", "GaussianRasterizationSettings"} <= set(api["renderer_imports"])
    for name in api["renderer_imports"]:
        assert getattr(dgr, name) is getattr(RZ, name), name
    # every GaussianRasterizationSettings(...) call: keywords == our NamedTuple fields (order irrelevant, all present)
    fields = set(RZ.GaussianRasterizationSettings._fields)
    assert len(api["settings_calls"]) >= 2
    for c in api["settings_calls"]:
        assert not c["args"] and set(c["keywords"]) == fields, set(c["keywords"]) ^ fields
    # GaussianRasterizer(raster_settings=...) and the forward call rasterizer(means3D=..., ...)
    assert "raster_settings" in inspect.signature(RZ.GaussianRasterizer.__init__).parameters
    fwd = set(inspect.signature(RZ.GaussianRasterizer.forward).parameters) - {"self"}
    assert len(api["rasterizer_calls"]) >= 1
    for kws in api["rasterizer_calls"]:
        assert set(kws) <= fwd and {"means3D", "means2D", "opacities"} <= set(kws), set(kws) - fwd
    # the reference unpacks exactly three outputs: rendered_image, radii, depth
    assert api["unpacks_image_radii_depth"]


def test_reference_scene_model_calls_apply_weights_with_our_slot_order(gold):
    import gaussianeditor_b200.rasterizer as RZ
    from gaussianeditor_b200 import gaussian_renderer as GR
    _, api = gold
    assert api["apply_weights_calls"] == [{"args": 10, "keywords": 0}]
    # positional slots of scene/gaussian_model.py:821-832 -> our parameter names
    ours = [p for p in inspect.signature(RZ.GaussianRasterizer.apply_weights).parameters if p != "self"]
    assert ours == ["means3D", "means2D", "opacities", "shs", "weights", "scales", "rotations", "cov3Ds_precomp", "cnt",
                    "image_weights"]
    # same as the reference package's own signatures (DGR/diff_gaussian_rasterization/__init__.py:311-322)
    assert "apply_weights" in api["rasterizer_methods"]
    for name, theirs in api["rasterizer_methods"].items():
        assert hasattr(RZ.GaussianRasterizer, name), name
        mine = [p for p in inspect.signature(getattr(RZ.GaussianRasterizer, name)).parameters if p != "self"]
        assert mine[:len(theirs)] == theirs, (name, mine, theirs)
    # the scene model imports these from the renderer module
    for name in api["model_imports_from_renderer"]:
        assert callable(getattr(GR, name)), name


def test_optimizer_surgery_equals_the_reference_functions(gold):
    from gaussianeditor_b200 import optim_surgery as OS
    z, _ = gold
    g, keep, ext = surgery_inputs()
    _, opt = bare_model()
    r = OS.prune_optimizer(opt, keep)
    assert all(isinstance(v, torch.nn.Parameter) and v.requires_grad for v in r.values())
    got = returned(r, "prune")
    got.update(snapshot(opt, "prune"))
    _assert_recorded(z, got, "prune")
    got = returned(OS.cat_tensors_to_optimizer(opt, {k: v.clone() for k, v in ext.items()}), "cat")   # :643-660
    got.update(snapshot(opt, "cat"))
    _assert_recorded(z, got, "cat")
    new_op = _normal(g, *opt.param_groups[3]["params"][0].shape)
    r = OS.replace_tensor_to_optimizer(opt, new_op.clone(), "opacity")                                 # reset_opacity
    assert r.keys() == {"opacity"}
    got = returned(r, "replace")
    got.update(snapshot(opt, "replace"))
    _assert_recorded(z, got, "replace")
    # and the optimizer keeps stepping like the reference's afterwards: one step of ours next to one step of an Adam
    # holding the reference's recorded state, in this process
    theirs = adam_from(z, "replace")
    adam_step(opt)
    adam_step(theirs)
    mine, want = snapshot(opt, "step"), snapshot(theirs, "step")
    assert sorted(mine) == sorted(want)
    for k in want:
        assert np.array_equal(mine[k], want[k]), k


@pytest.mark.parametrize("deg", PLY_DEGREES)
def test_ply_bytes_equal_what_the_reference_writer_hands_to_plyfile(gold, tmp_path, deg):
    from gaussianeditor_b200 import ply_io
    z, api = gold
    names = api["ply_fields"][str(deg)]
    table = z[f"ply/{deg}"]                                # the REFERENCE's vertex table, fields in its order
    assert table.shape[1] == len(names)
    p, _ = bare_model(P=11, deg=deg, seed=deg)
    ours = str(tmp_path / "ours.ply")
    ply_io.write_gaussian_ply(ours, xyz=p["xyz"].detach().numpy(), features_dc=p["f_dc"].detach().numpy(),
                              features_rest=p["f_rest"].detach().numpy(), opacity=p["opacity"].detach().numpy(),
                              scaling=p["scaling"].detach().numpy(), rotation=p["rotation"].detach().numpy())
    raw = open(ours, "rb").read()
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % len(table) +
              "".join(f"property float {n}\n" for n in names) + "end_header\n").encode()   # plyfile's header
    assert raw[:len(header)] == header
    assert raw[len(header):] == np.ascontiguousarray(table, "<f4").tobytes()   # body: bit for bit the reference's table
    # what the reference's load_ply (:447-501) reads by name comes back from our reader unchanged
    cols = ply_io.read_vertex_table(ours)
    assert list(cols) == names
    for i, n in enumerate(names):
        assert np.array_equal(np.asarray(cols[n], np.float32).ravel(), table[:, i]), n
