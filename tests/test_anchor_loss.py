"""GaussianEditor's anchor loss on the CUDA kernels (``gaussianeditor_b200.anchor_loss``, ``csrc/anchor_loss.cu``).

CPU: the C ABI and its argument checks, the Python entry's checks, no float atomics in the kernels, the harness's torch
restatement against the reference's own function (tests/golden/anchor, made by tools/make_anchor_golden.py) and its
generation / schedule bookkeeping. GPU: values and gradients against an fp64 truth and against the golden fixture,
bit-reproducibility, CUDA-graph capture, no host synchronisation, out-of-range generations, and the edit loop."""
import functools
import json
import math
import os
import re
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gaussianeditor_b200 import _lib
from gaussianeditor_b200.anchor_loss import KEYS, TERMS

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "gsr_b200.h")
GOLDEN = os.path.join(HERE, "golden", "anchor", "reference_anchor.npz")
ENTRY = ("gsr_anchor_loss_forward", "gsr_anchor_loss_backward")
EPS = 2.0 ** -24


def _bits(t):
    return t.contiguous().view(torch.int32)


def _shapes(P, deg):
    return {"_xyz": (P, 3), "_features_dc": (P, 1, 3), "_features_rest": (P, (deg + 1) ** 2 - 1, 3),
            "_scaling": (P, 3), "_rotation": (P, 4), "_opacity": (P, 1)}


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_symbols_declared_exported_and_bound():
    header = open(HEADER).read()
    lib = _lib.load()
    for name in ("gsr_anchor_loss_scratch_bytes",) + ENTRY:
        assert re.search(rf"GSR_API \w+ {name}\(", header), name
        assert name in _lib.SYMBOLS and hasattr(lib, name)
        assert getattr(lib, name).argtypes
    assert lib.gsr_abi_version() == 2
    assert lib.gsr_anchor_loss_scratch_bytes(1) < lib.gsr_anchor_loss_scratch_bytes(10_000_000) < 1 << 20


def _terms(**field):
    arr = (_lib.AnchorTerm * 6)()
    for d in arr:   # fake but non-NULL pointers: every case below must be rejected before they are used
        d.p = d.a = d.g = 256
        d.D = 3
    for k, val in field.items():
        setattr(arr[0], k, val)
    return arr


BAD = {
    "null_terms": ({}, dict(terms=None)), "null_p": (dict(p=None), {}), "null_a": (dict(a=None), {}),
    "null_g": (dict(g=None), {}), "P_negative": ({}, dict(P=-1)), "D_negative": (dict(D=-1), {}),
    "D_huge": (dict(D=(1 << 24) + 1), {}), "no_schedule": ({}, dict(n_schedule=0)),
    "null_schedule": ({}, dict(schedule=None)), "null_mask": ({}, dict(mask=None)),
    "null_generation": ({}, dict(generation=None)), "null_scratch": ({}, dict(scratch=None)),
    "small_scratch": ({}, dict(scratch_bytes=8)), "null_out": ({}, dict(out=None)),
}


@pytest.mark.parametrize("entry", ENTRY)
@pytest.mark.parametrize("case", sorted(BAD))
def test_entry_points_reject_invalid_arguments_before_the_device(entry, case):
    lib = _lib.load()
    field, call = BAD[case]
    if case == "null_g" and entry == "gsr_anchor_loss_forward":
        pytest.skip("the forward does not read g")
    P = call.get("P", 1000)
    args = dict(terms=_terms(**field), P=P, mask=512, generation=768, schedule=1024, n_schedule=3, scratch=2048,
                scratch_bytes=lib.gsr_anchor_loss_scratch_bytes(max(P, 0)), out=4096)
    args.update(call)
    rc = getattr(lib, entry)(args["terms"], args["P"], args["mask"], args["generation"], args["schedule"],
                             args["n_schedule"], args["scratch"], args["scratch_bytes"], args["out"], None)
    assert rc == -1, case
    assert lib.gsr_last_error().decode().startswith(entry), lib.gsr_last_error()


def _model(P=5, deg=1, device="cpu", seed=0):
    g = torch.Generator().manual_seed(seed)
    m = SimpleNamespace()
    for k, s in _shapes(P, deg).items():
        setattr(m, k, torch.randn(s, generator=g).to(device).requires_grad_(True))
    m.anchor = {k: getattr(m, k).detach().clone() for k in TERMS}
    m.mask = (torch.arange(P) % 2 == 0).to(device)
    m._generation = torch.zeros(P, dtype=torch.int64, device=device)
    m._anchor_loss_schedule = torch.tensor([0.01], device=device)
    return m


def _bad_models():
    yield "float32", lambda m: setattr(m, "_xyz", m._xyz.double())
    yield "float32", lambda m: m.anchor.update(_scaling=m.anchor["_scaling"].half())
    yield "int64", lambda m: setattr(m, "_generation", m._generation.int())
    yield "float32", lambda m: setattr(m, "_anchor_loss_schedule", m._anchor_loss_schedule.double())
    yield "shape", lambda m: m.anchor.update(_rotation=m.anchor["_rotation"][:, :3].contiguous())
    yield "shape", lambda m: setattr(m, "_opacity", m._opacity[:4])
    yield "shape", lambda m: setattr(m, "_generation", m._generation[:4])
    yield "at least one", lambda m: setattr(m, "_anchor_loss_schedule", m._anchor_loss_schedule[:0])
    yield "contiguous", lambda m: setattr(m, "_xyz", torch.zeros(3, 5).t())
    yield "contiguous", lambda m: m.anchor.update(_features_dc=torch.zeros(5, 1, 6)[:, :, ::2])
    yield "bool", lambda m: setattr(m, "mask", m.mask.to(torch.uint8))
    yield "bool", lambda m: setattr(m, "mask", m.mask.float())
    yield "exactly", lambda m: m.anchor.pop("_opacity")
    yield "exactly", lambda m: m.anchor.update(_extra=m.anchor["_xyz"])
    yield "CUDA", lambda m: None


@pytest.mark.parametrize("i", range(len(list(_bad_models()))))
def test_python_entry_rejects_bad_inputs(i):
    from gaussianeditor_b200 import anchor_loss
    match, spoil = list(_bad_models())[i]
    m = _model()
    spoil(m)
    with pytest.raises(ValueError, match=match):
        anchor_loss(m)


def test_empty_anchor_returns_the_reference_zeros():
    from gaussianeditor_b200 import anchor_loss
    m = _model()
    m.anchor = {}
    assert anchor_loss(m) == {k: 0 for k in KEYS}


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="cuobjdump is not available")
def test_anchor_kernels_have_no_float_atomics():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels, name = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            name = m.group(1)
            kernels[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            kernels[name].append(line.split("*/", 1)[1].split(";")[0].strip())
    ours = {n: b for n, b in kernels.items() if re.search(r"anchor_(fwd|finish|bwd)_kernel", n)}
    assert len(ours) == 3, sorted(ours)
    fatom = re.compile(r"^(?:@!?U?P\w+\s+)?(RED|ATOM)[GS]?\.\S*\.F(16|32|64)")
    for n, body in ours.items():
        assert body and not [i for i in body if fatom.match(i)], n


def _golden():
    z = np.load(GOLDEN)
    return z, json.loads(str(z["meta"]))


def _golden_model(z, case, device):
    from gaussianeditor_b200.edit_loop import EditScene
    m = EditScene.__new__(EditScene)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    for k in TERMS:
        setattr(m, k, t(z[f"{case}/param/{k}"]).requires_grad_(True))
    m.anchor = {k: t(z[f"{case}/anchor/{k}"]) for k in TERMS}
    m.mask = t(z[f"{case}/mask"])
    m._generation = t(z[f"{case}/generation"])
    m._anchor_loss_schedule = t(z[f"{case}/schedule"])
    return m


def _backward(m, out, lam):
    loss = 0
    for k, v in out.items():
        loss = loss + v * lam[k]
    loss.backward()
    return {k: getattr(m, k).grad.detach().cpu() for k in TERMS}


def _same_nan_and_close(got, ref, rtol, atol=0.0):
    got, ref = torch.as_tensor(got, dtype=torch.float64), torch.as_tensor(ref, dtype=torch.float64)
    assert torch.equal(torch.isnan(got), torch.isnan(ref))
    ok = ~torch.isnan(ref)
    err = (got[ok] - ref[ok]).abs()
    bound = rtol * ref[ok].abs() + atol
    assert bool((err <= bound).all()), float((err - bound).max())


def test_torch_restatement_matches_the_reference_golden():
    z, meta = _golden()
    assert len(meta["cases"]) == 18 and meta["keys"] == list(KEYS)
    nan_cases = 0
    for case in meta["cases"]:
        m = _golden_model(z, case, "cpu")
        out = m.anchor_loss_torch()
        assert list(out) == list(KEYS)
        vals = torch.stack([out[k].detach() for k in KEYS])
        _same_nan_and_close(vals, z[f"{case}/out"], 1e-6)
        nan_cases += bool(torch.isnan(vals).any())
        grads = _backward(m, out, meta["lambda"])
        for k in TERMS:
            _same_nan_and_close(grads[k], z[f"{case}/grad/{k}"], 1e-6, 1e-30)
    assert nan_cases >= 6   # the empty masks and degree 0


def test_harness_generation_and_schedule_bookkeeping():
    from gaussianeditor_b200 import synth
    from gaussianeditor_b200.edit_loop import EditScene
    cloud, _ = synth.make_config("c5", P=400)
    scene = EditScene(cloud, "cpu", track_anchor=True)
    assert EditScene(cloud, "cpu").anchor == {}
    f = np.float32
    expected = [f(0.01)]
    assert torch.equal(scene._anchor_loss_schedule, torch.tensor(expected))
    assert torch.equal(scene._generation, torch.zeros(400, dtype=torch.int64))
    for gen in (1, 2, 3):
        P = scene._xyz.shape[0]
        scene.xyz_gradient_accum = torch.rand(P, 1, generator=torch.Generator().manual_seed(gen))
        scene.denom = torch.ones(P, 1)
        scene.densify_and_prune()
        n = scene._xyz.shape[0]
        k = max(1, int(P * 0.01))
        # clones are appended with the new generation; kept rows keep theirs
        assert torch.equal(scene._generation[n - k:], torch.full((k,), gen))
        assert bool((scene._generation[: n - k] < gen).all())
        assert scene._generation.shape == scene.mask.shape == (n,)
        # update_anchor_loss_schedule, by hand in fp32
        expected = [min(f(w * f(1.3)), f(10)) for w in expected]
        if len(expected) > 1:
            assert expected[-1] == 0
            expected[-1] = f(0.01)
        expected.append(f(0))
        assert torch.equal(scene._anchor_loss_schedule, torch.tensor(expected, dtype=torch.float32)), gen
        for k_ in TERMS:   # re-anchored on the new rows
            assert torch.equal(scene.anchor[k_], getattr(scene, k_).detach())
    f13 = f(1.3)
    assert expected == [f(f(f(f(0.01) * f13) * f13) * f13), f(f(0.01) * f13), f(0.01), f(0)]


def test_edit_loop_rejects_a_synchronising_anchor_in_the_fixed_step():
    from gaussianeditor_b200.edit_loop import run_edit_loop
    for kw in (dict(cuda_graph=True), dict(static_capacity=True)):
        with pytest.raises(ValueError, match="anchor"):
            run_edit_loop(None, steps=1, P=100, anchor="torch", **kw)
    with pytest.raises(ValueError, match="anchor"):
        run_edit_loop(None, steps=1, P=100, anchor="fused")


# ---------------------------------------------------------------------------------------------------------------- GPU
SCHEDULE = [0.02197, 0.0169, 0.0, 0.01, 0.0]   # zero weights in the middle and at the newborn end
LAM = dict(zip(KEYS, (5.0, 50.0, 50.0, 50.0)))


def _gpu_model(P, deg, mask_kind, seed=0, nan_unedited=False):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    m = SimpleNamespace()
    for k, s in _shapes(P, deg).items():
        a = torch.randn(s, generator=gen, device="cuda")
        p = a + 0.1 * torch.randn(s, generator=gen, device="cuda")
        setattr(m, k, p)
        m.anchor = getattr(m, "anchor", {})
        m.anchor[k] = a
    if mask_kind == "random":
        mask = torch.rand(P, generator=gen, device="cuda") < 0.2
    elif mask_kind == "spatial":
        d = m._xyz.norm(dim=1)
        mask = d <= torch.quantile(d[: min(P, 1_000_000)], 0.2)
    elif mask_kind == "all":
        mask = torch.ones(P, dtype=torch.bool, device="cuda")
    elif mask_kind == "empty":
        mask = torch.zeros(P, dtype=torch.bool, device="cuda")
    else:   # single row
        mask = torch.zeros(P, dtype=torch.bool, device="cuda")
        mask[P // 2] = True
    m.mask = mask
    if nan_unedited:
        for k in TERMS:
            getattr(m, k)[~mask] = float("nan")
            m.anchor[k][~mask] = float("nan")
    for k in TERMS:
        getattr(m, k).requires_grad_(True)
    m._generation = torch.randint(0, len(SCHEDULE), (P,), generator=gen, device="cuda")
    m._anchor_loss_schedule = torch.tensor(SCHEDULE, device="cuda")
    return m


def _truth(m, grad_out):
    """fp64: the four values and the six gradients for grad_out = (color, geo, opacity, scale)."""
    mask = m.mask
    N = float(mask.sum())
    w = m._anchor_loss_schedule.double()[m._generation]
    L, G = {}, {}
    for k in TERMS:
        p, a = getattr(m, k).detach().double(), m.anchor[k].double()
        P = p.shape[0]
        D = math.prod(p.shape[1:])
        d = (p - a).reshape(P, D)
        wm = w[:, None]
        sq = torch.where(mask[:, None], wm * d * d, torch.zeros((), dtype=torch.float64, device=d.device))
        L[k] = float(sq.sum()) / (N * D) if N * D > 0 else math.nan
        group = {"_xyz": 1, "_rotation": 1, "_features_dc": 0, "_features_rest": 0, "_opacity": 2, "_scaling": 3}[k]
        g = 2 * d * (grad_out[group] / (N * D) if N * D > 0 else 0.0) * wm
        G[k] = torch.where(mask[:, None], g, torch.zeros((), dtype=torch.float64, device=d.device)).reshape(p.shape)
    vals = [L["_features_dc"] + L["_features_rest"], L["_xyz"] + L["_rotation"], L["_opacity"], L["_scaling"]]
    return vals, G


def _run(m):
    from gaussianeditor_b200 import anchor_loss
    for k in TERMS:
        getattr(m, k).grad = None
    out = anchor_loss(m)
    vals = torch.stack([out[k].detach() for k in KEYS]).cpu()
    grads = _backward(m, out, LAM)
    return vals, grads


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 31, 32, 33, 1000, 100_000, 1_000_000])
@pytest.mark.parametrize("deg", [3, 0])
@pytest.mark.parametrize("mask_kind", ["random", "spatial", "all", "empty", "single"])
def test_against_fp64_truth(P, deg, mask_kind):
    m = _gpu_model(P, deg, mask_kind, seed=P + deg, nan_unedited=mask_kind in ("random", "single"))
    vals, grads = _run(m)
    tv, tg = _truth(m, list(LAM.values()))
    n_edit = int(m.mask.sum())
    for i in range(4):
        if math.isnan(tv[i]):
            assert math.isnan(float(vals[i])), (i, vals)
        else:
            assert abs(float(vals[i]) - tv[i]) <= 8 * EPS * abs(tv[i]), (i, float(vals[i]), tv[i])
    assert math.isnan(float(vals[0])) == (deg == 0 or n_edit == 0)
    un = (~m.mask).cpu()
    for k in TERMS:
        g, g64 = grads[k].double(), tg[k].cpu()
        assert bool(((g - g64).abs() <= 8 * EPS * g64.abs() + 2.0 ** -149).all()), k
        assert not bool(torch.any(_bits(grads[k][un]))), k   # +0.0 bit for bit, even over NaN p and a


@pytest.mark.gpu
def test_against_the_reference_golden():
    z, meta = _golden()
    from gaussianeditor_b200 import anchor_loss
    for case in meta["cases"]:
        m = _golden_model(z, case, "cuda")
        out = anchor_loss(m)
        vals = torch.stack([out[k].detach() for k in KEYS]).cpu()
        _same_nan_and_close(vals, z[f"{case}/out"], 1e-6)
        grads = _backward(m, out, meta["lambda"])
        for k in TERMS:
            _same_nan_and_close(grads[k], z[f"{case}/grad/{k}"], 16 * EPS, 2.0 ** -149)


@pytest.mark.gpu
def test_reproducible_capturable_and_sync_free():
    from gaussianeditor_b200 import anchor_loss
    m = _gpu_model(300_000, 3, "spatial", seed=5)
    v1, g1 = _run(m)
    v2, g2 = _run(m)
    assert torch.equal(_bits(v1), _bits(v2))
    for k in TERMS:
        assert torch.equal(_bits(g1[k]), _bits(g2[k])), k
    # forward + backward in a CUDA graph replays to the eager bits
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _run(m)   # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(side)
    for k in TERMS:
        getattr(m, k).grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = anchor_loss(m)
        cap_vals = torch.stack([out[k] for k in KEYS]).detach()
        loss = sum(out[k] * LAM[k] for k in KEYS)
        loss.backward()
    for k in TERMS:
        getattr(m, k).grad.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(cap_vals.cpu()), _bits(v1))
    for k in TERMS:
        assert torch.equal(_bits(getattr(m, k).grad.cpu()), _bits(g1[k])), k
    # eager forward + backward with no host synchronisation
    for k in TERMS:
        getattr(m, k).grad = None
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = anchor_loss(m)
        sum(out[k] * LAM[k] for k in KEYS).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")


@pytest.mark.gpu
def test_rejects_tensors_off_the_mask_device():
    from gaussianeditor_b200 import anchor_loss
    for attr in ("_scaling", "_generation"):
        m = _model(device="cuda")
        setattr(m, attr, getattr(m, attr).detach().cpu())
        with pytest.raises(ValueError, match="device"):
            anchor_loss(m)
    m = _model(device="cuda")
    m.anchor["_opacity"] = m.anchor["_opacity"].cpu()
    with pytest.raises(ValueError, match="device"):
        anchor_loss(m)


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [-1, len(SCHEDULE), 1 << 40])
def test_out_of_range_generation_gives_nan_and_no_fault(bad):
    m = _gpu_model(1000, 3, "all", seed=9)
    m._generation[17] = bad
    vals, grads = _run(m)
    torch.cuda.synchronize()
    assert bool(torch.isnan(vals).all())
    for k in TERMS:
        assert bool(torch.isnan(grads[k][17]).all()), k
        assert bool(torch.isfinite(grads[k][18:]).all()), k


def _edit_loop(anchor, cuda_graph=False, **kw):
    from gaussianeditor_b200.edit_loop import run_edit_loop
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    return run_edit_loop(functools.partial(GaussianRasterizer, deterministic=True), steps=300, P=50_000,
                         densification_interval=100, deterministic=True, anchor=anchor, cuda_graph=cuda_graph, **kw)


@pytest.mark.gpu
def test_edit_loop_torch_and_kernel_arms_agree():
    a = _edit_loop("torch")
    b = _edit_loop("kernel")
    assert a["counts"] == b["counts"] and len(set(a["counts"])) > 1
    assert torch.equal(a["generation"], b["generation"]) and int(a["generation"].max()) == 2
    assert torch.equal(a["anchor_schedule"], b["anchor_schedule"]) and a["anchor_schedule"].numel() == 3
    for x, y in zip(a["losses"], b["losses"]):
        assert abs(x - y) <= 1e-3 * abs(x), (x, y)
    base = _edit_loop(None)
    assert "generation" not in base
    assert any(abs(x - y) > 0 for x, y in zip(base["losses"], a["losses"]))   # the term is in the loss


@pytest.mark.gpu
def test_edit_loop_kernel_arm_in_the_captured_step():
    kw = dict(grad_mask="kernel", optimizer="masked")
    eager = _edit_loop("kernel", **kw)
    graph = _edit_loop("kernel", cuda_graph=True, **kw)
    assert graph["counts"] == eager["counts"] and len(set(graph["counts"])) > 1
    assert torch.equal(graph["generation"], eager["generation"])
    assert torch.equal(graph["anchor_schedule"], eager["anchor_schedule"])
    with pytest.raises(ValueError, match="anchor"):
        _edit_loop("torch", cuda_graph=True)
