"""Record what the reference's own callers of the rasterizer do, for tests/test_reference_callers.py:

    python tools/make_caller_golden.py <GaussianEditor checkout> tests/golden/callers/reference_callers.npz

The reference's gaussian_renderer and scene/gaussian_model modules are imported unchanged, with
``diff_gaussian_rasterization`` resolving to this repository's drop-in package and the two third-party modules absent
here (``plyfile``, ``simple_knn``) stubbed. Recorded: the names, keywords and positional slots the reference uses on
the rasterizer (read from its source), the parameters / returned tensors / Adam state after its optimizer surgery, and
the vertex table its save_ply hands to plyfile. CPU only."""
import ast
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_reference_callers as T   # noqa: E402


class _Captured:
    def __init__(self, data, name):
        self.data, self.name = data, name


def install_stubs():
    ply = types.ModuleType("plyfile")

    class PlyElement:
        @staticmethod
        def describe(data, name):
            return _Captured(data, name)

    class PlyData:
        last_written = None

        def __init__(self, elements):
            self.elements = elements

        def write(self, path):
            PlyData.last_written = (path, self.elements)
    ply.PlyElement, ply.PlyData = PlyElement, PlyData
    knn = types.ModuleType("simple_knn")
    knn_c = types.ModuleType("simple_knn._C")
    knn_c.distCUDA2 = lambda pts: torch.full((pts.shape[0],), 1e-2)
    knn._C = knn_c
    sys.modules.update({"plyfile": ply, "simple_knn": knn, "simple_knn._C": knn_c})
    return ply


def calls(tree, pred):
    return [n for n in ast.walk(tree) if isinstance(n, ast.Call) and pred(n.func)]


def imports_from(tree, module_suffix):
    return sorted(a.name for n in ast.walk(tree) if isinstance(n, ast.ImportFrom) and (n.module or "").endswith(module_suffix)
                  for a in n.names)


def model_with(GM, params, opt, deg):
    m = GM.GaussianModel.__new__(GM.GaussianModel)
    m.setup_functions()
    m.active_sh_degree = m.max_sh_degree = deg
    m._xyz, m._features_dc, m._features_rest = params["xyz"], params["f_dc"], params["f_rest"]
    m._opacity, m._scaling, m._rotation = params["opacity"], params["scaling"], params["rotation"]
    m.optimizer = opt
    return m


def main(ref_root, out):
    sys.path.insert(0, ref_root)
    ply = install_stubs()
    import diff_gaussian_rasterization as dgr
    assert os.path.dirname(dgr.__file__).startswith(ROOT), "the reference must resolve the drop-in, not its own package"
    import gaussiansplatting.scene.gaussian_model as GM
    gs = os.path.join(ref_root, "gaussiansplatting")
    rsrc = open(os.path.join(gs, "gaussian_renderer", "__init__.py")).read()
    rtree = ast.parse(rsrc)
    mtree = ast.parse(open(os.path.join(gs, "scene", "gaussian_model.py")).read())
    dtree = ast.parse(open(os.path.join(gs, "submodules", "diff-gaussian-rasterization", "diff_gaussian_rasterization",
                                        "__init__.py")).read())
    cls = next(n for n in ast.walk(dtree) if isinstance(n, ast.ClassDef) and n.name == "GaussianRasterizer")
    aw = calls(mtree, lambda f: isinstance(f, ast.Attribute) and f.attr == "apply_weights" and
               isinstance(f.value, ast.Name) and f.value.id == "rasterizer")
    api = {
        "renderer_imports": imports_from(rtree, "diff_gaussian_rasterization"),
        "settings_calls": [{"args": len(c.args), "keywords": sorted(k.arg for k in c.keywords)}
                           for c in calls(rtree, lambda f: isinstance(f, ast.Name) and f.id == "GaussianRasterizationSettings")],
        "rasterizer_calls": [sorted(k.arg for k in c.keywords)
                             for c in calls(rtree, lambda f: isinstance(f, ast.Name) and f.id == "rasterizer")],
        "unpacks_image_radii_depth": "rendered_image, radii, depth = rasterizer(" in rsrc,
        "apply_weights_calls": [{"args": len(c.args), "keywords": len(c.keywords)} for c in aw],
        "rasterizer_methods": {fn.name: [a.arg for a in fn.args.args if a.arg != "self"]
                               for fn in cls.body if isinstance(fn, ast.FunctionDef) and not fn.name.startswith("__")},
        "model_imports_from_renderer": imports_from(mtree, "gaussian_renderer"),
        "ply_fields": {},
    }
    rec = {}
    g, keep, ext = T.surgery_inputs()
    params, opt = T.bare_model()
    m = model_with(GM, params, opt, 2)
    rec.update(T.returned(m._prune_optimizer(keep), "prune")); rec.update(T.snapshot(opt, "prune"))
    rec.update(T.returned(m.cat_tensors_to_optimizer({k: v.clone() for k, v in ext.items()}), "cat"))
    rec.update(T.snapshot(opt, "cat"))
    new_op = T._normal(g, *opt.param_groups[3]["params"][0].shape)
    rec.update(T.returned(m.replace_tensor_to_optimizer(new_op.clone(), "opacity"), "replace"))
    rec.update(T.snapshot(opt, "replace"))
    for deg in T.PLY_DEGREES:
        params, opt = T.bare_model(P=11, deg=deg, seed=deg)
        m = model_with(GM, params, opt, deg)
        with tempfile.TemporaryDirectory() as tmp:   # save_ply creates the directory; the stub writes nothing
            m.save_ply(os.path.join(tmp, "point_cloud.ply"))
        _, elements = ply.PlyData.last_written
        table = elements[0].data
        api["ply_fields"][str(deg)] = list(table.dtype.names)
        rec[f"ply/{deg}"] = np.stack([table[n] for n in table.dtype.names], axis=1).astype("<f4")
    np.savez_compressed(out, api=np.array(json.dumps(api, sort_keys=True)), **rec)
    print("wrote", out, len(rec), "arrays")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
