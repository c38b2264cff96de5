"""``MaskedAdam`` / ``gsr_adam_masked``: torch's Adam restricted to the Gaussians under edit, one launch per step.

CPU: the entry point is declared and exported, rejects every invalid argument before touching a device, the optimizer
rejects the options, dtypes and shapes it does not implement, a ``torch.optim.Adam`` state dict moves into it and back
unchanged, ``optim_surgery`` prunes and extends its state, and its kernels contain no RED/ATOM.
GPU: one step from random state on every Gaussian width, a degree-0 cloud and a lone D = 1 group, at P from 1 to 500k,
under random, spatial, full, empty and single-row masks: unedited rows keep their bits even holding NaN, edited rows are
within 1 ulp(p) + 4 ulp(update) of an fp64 Adam (2 ulp for the moments), a bound torch's foreach and fused Adam are held
to on the same inputs. lr changes and groups without gradient behave as in torch. A 50-step trajectory under the edit
invariant matches torch's Adam (unedited rows bit for bit), is reproducible, and freezes a row dropped from the mask.
A capturable step replays in a CUDA graph bit for bit and runs eagerly without a host synchronisation. The edit-loop
harnesses (single GPU, eager and graphed, and sharded at world 1 across a rebalance) with optimizer="masked" keep the
Adam arm's counts, its unedited rows bit for bit, and its losses within 1e-3.
"""
import functools
import math
import os
import re
import shutil
import socket
import subprocess

import pytest
import torch
import torch.distributed as dist

from gaussianeditor_b200 import MaskedAdam, _lib, optim_surgery

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "gsr_b200.h")
SHAPES = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
LRS = {"xyz": 1.6e-5, "f_dc": 2.5e-3, "f_rest": 1.25e-4, "opacity": 0.1, "scaling": 1e-2, "rotation": 2e-3}
LAYOUTS = {"six": SHAPES, "deg0": dict(SHAPES, f_rest=(0, 3)), "d1": {"opacity": (1,)}}


def _bits(t):
    return t.contiguous().view(torch.int32)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_symbol_declared_and_exported():
    header = open(HEADER).read()
    assert re.search(r"GSR_API int gsr_adam_masked\(", header)
    assert "gsr_adam_masked" in _lib.SYMBOLS and hasattr(_lib.load(), "gsr_adam_masked")
    assert _lib.load().gsr_abi_version() == 2


def _desc(n=1, **field):
    arr = (_lib.AdamGroup * max(n, 1))()
    for d in arr:   # fake but non-NULL pointers: every case below must be rejected before they are used
        d.p = d.g = d.m = d.v = 256
        d.D, d.lr, d.beta1, d.beta2, d.eps, d.step = 3, 1e-3, 0.9, 0.999, 1e-8, 1.0
    for k, val in field.items():
        setattr(arr[0], k, val)
    return arr


BAD = {
    "null_p": (dict(p=None), {}), "null_g": (dict(g=None), {}), "null_m": (dict(m=None), {}),
    "null_v": (dict(v=None), {}), "null_mask": ({}, dict(mask=None)), "null_groups": ({}, dict(groups=None)),
    "P_negative": ({}, dict(P=-1)), "D_negative": (dict(D=-1), {}), "D_huge": (dict(D=(1 << 24) + 1), {}),
    "no_groups": ({}, dict(n=0)), "too_many_groups": ({}, dict(n=17)), "beta1_one": (dict(beta1=1.0), {}),
    "beta1_negative": (dict(beta1=-0.1), {}), "beta2_one": (dict(beta2=1.0), {}), "beta2_nan": (dict(beta2=math.nan), {}),
    "eps_negative": (dict(eps=-1e-8), {}), "step_zero": (dict(step=0.0), {}),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_entry_point_rejects_invalid_arguments_before_the_device(case):
    lib = _lib.load()
    field, call = BAD[case]
    n = call.get("n", 1)
    arr = _desc(n if 0 < n <= 16 else 1, **field)
    groups = call["groups"] if "groups" in call else arr
    mask = call["mask"] if "mask" in call else 512
    rc = lib.gsr_adam_masked(groups, n, call.get("P", 1000), mask, None)
    assert rc == -1, case
    assert lib.gsr_last_error().decode().startswith("gsr_adam_masked"), lib.gsr_last_error()


def _groups(P=6, device="cpu", shapes=SHAPES, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [{"params": [torch.nn.Parameter(torch.randn((P,) + s, generator=g).to(device))], "lr": LRS[n], "name": n}
            for n, s in shapes.items()]


@pytest.mark.parametrize("kw", [dict(weight_decay=0.1), dict(amsgrad=True), dict(maximize=True), dict(foreach=True),
                                dict(fused=True), dict(lr=torch.tensor(1e-3)), dict(betas=(1.0, 0.999)),
                                dict(eps=-1.0), dict(lr=-1.0)])
def test_constructor_rejects_unsupported_options(kw):
    with pytest.raises(ValueError):
        MaskedAdam(_groups(), **kw)


def test_constructor_rejects_params_and_masks_it_cannot_step():
    with pytest.raises(ValueError, match="float32"):
        MaskedAdam([torch.nn.Parameter(torch.zeros(4, 3, dtype=torch.float64))])
    with pytest.raises(ValueError, match="contiguous"):
        MaskedAdam([torch.zeros(3, 4).t()])
    with pytest.raises(ValueError, match="exactly one"):
        MaskedAdam([torch.nn.Parameter(torch.zeros(4, 3)), torch.nn.Parameter(torch.zeros(4, 1))])
    with pytest.raises(TypeError):
        MaskedAdam(_groups(), nesterov=True)
    opt = MaskedAdam(_groups())
    with pytest.raises(ValueError, match="bool or uint8"):
        opt.set_mask(torch.ones(6))
    with pytest.raises(ValueError, match="1-D"):
        opt.set_mask(torch.ones(2, 3, dtype=torch.bool))
    with pytest.raises(ValueError, match="CUDA"):
        opt.set_mask(torch.ones(6, dtype=torch.bool))
    with pytest.raises(RuntimeError, match="set_mask"):
        opt.step()
    opt.param_groups[0]["lr"] = torch.tensor(0.1)   # a tensor lr written into a group is caught at the step
    opt._mask = torch.ones(6, dtype=torch.uint8)
    with pytest.raises(ValueError, match="float lr"):
        opt.step()


def _adam_cpu_state():
    groups = _groups(P=7)
    adam = torch.optim.Adam(groups, eps=1e-15)
    for k in range(3):
        for i, gr in enumerate(adam.param_groups):
            p = gr["params"][0]
            p.grad = None if (k == 1 and i == 2) else torch.randn_like(p)
        adam.step()
    return adam


def _same_state_dict(a, b):
    assert a["param_groups"] == b["param_groups"]
    assert a["state"].keys() == b["state"].keys()
    for k in a["state"]:
        assert a["state"][k].keys() == b["state"][k].keys()
        for key in a["state"][k]:
            x, y = a["state"][k][key], b["state"][k][key]
            assert x.dtype == y.dtype and x.device == y.device and torch.equal(x, y), (k, key)


def test_state_dict_round_trip_with_torch_adam():
    adam = _adam_cpu_state()
    sd = adam.state_dict()
    ours = MaskedAdam(_groups(P=7), eps=1e-15)
    ours.load_state_dict(sd)
    _same_state_dict(ours.state_dict(), sd)
    back = torch.optim.Adam(_groups(P=7), eps=1e-15)
    back.load_state_dict(ours.state_dict())
    _same_state_dict(back.state_dict(), sd)
    assert all(st["step"].dtype == torch.float32 and st["step"].device.type == "cpu" for st in ours.state.values())
    assert ours.state[ours.param_groups[2]["params"][0]]["step"].item() == 2.0   # no grad at the second step


def test_optim_surgery_on_its_state():
    sd = _adam_cpu_state().state_dict()
    ours = MaskedAdam(_groups(P=7), eps=1e-15)
    ours.load_state_dict(sd)
    before = {g["name"]: dict(ours.state[g["params"][0]]) for g in ours.param_groups}
    keep = torch.tensor([True, False, True, True, False, True, True])
    optim_surgery.prune_optimizer(ours, keep)
    ext = {n: torch.randn((2,) + s) for n, s in SHAPES.items()}
    optim_surgery.cat_tensors_to_optimizer(ours, ext)
    for g in ours.param_groups:
        p, st, old = g["params"][0], ours.state[g["params"][0]], before[g["name"]]
        assert p.shape[0] == 7 and isinstance(p, torch.nn.Parameter)
        assert torch.equal(p.detach()[5:], ext[g["name"]])
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(st[key][:5], old[key][keep]) and not st[key][5:].any(), (g["name"], key)
        assert torch.equal(st["step"], old["step"])


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="cuobjdump is not available")
def test_masked_adam_kernels_have_no_atomics():
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
    ours = {n: b for n, b in kernels.items() if "adam_masked_kernel" in n or "adam_step_kernel" in n}
    assert len(ours) == 2, sorted(ours)
    atom = re.compile(r"^(?:@!?U?P\w+\s+)?(RED|ATOM)")
    for n, body in ours.items():
        assert body and not [i for i in body if atom.match(i)], n


# ---------------------------------------------------------------------------------------------------------------- GPU
def _mask(kind, P, pos, gen):
    if kind == "random20":
        return torch.rand(P, generator=gen, device="cuda") < 0.2
    if kind == "spatial20":
        d = pos.norm(dim=1)
        return d <= torch.quantile(d, 0.2)
    if kind == "all":
        return torch.ones(P, dtype=torch.bool, device="cuda")
    if kind == "none":
        return torch.zeros(P, dtype=torch.bool, device="cuda")
    m = torch.zeros(P, dtype=torch.bool, device="cuda")
    m[P // 2] = True
    return m


def _inputs(P, shapes, seed):
    """Random fp32 state per group: p, g, m and v >= 0 (a state reached after a few steps)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for n, s in shapes.items():
        sh = (P,) + s
        out.append(dict(name=n, p=torch.randn(sh, generator=gen, device="cuda"),
                        g=torch.randn(sh, generator=gen, device="cuda") * 1e-2,
                        m=torch.randn(sh, generator=gen, device="cuda") * 1e-3,
                        v=torch.rand(sh, generator=gen, device="cuda") * 1e-4))
    return out, gen


def _make(kind, tensors, step0, mask=None, capturable=False):
    params = [torch.nn.Parameter(t["p"].clone()) for t in tensors]
    for p, t in zip(params, tensors):
        p.grad = t["g"].clone()
    groups = [{"params": [p], "lr": LRS[t["name"]], "name": t["name"]} for p, t in zip(params, tensors)]
    if kind == "masked":
        opt = MaskedAdam(groups, eps=1e-15, mask=mask, capturable=capturable)
    else:
        opt = torch.optim.Adam(groups, eps=1e-15, foreach=(kind == "foreach"), fused=(kind == "fused"),
                               capturable=capturable)
    on_dev = kind == "fused" or capturable
    for p, t in zip(params, tensors):
        step = torch.tensor(float(step0), dtype=torch.float32, device="cuda" if on_dev else "cpu")
        opt.state[p] = {"step": step, "exp_avg": t["m"].clone(), "exp_avg_sq": t["v"].clone()}
    return opt, params


def _ulp(x):
    a = x.abs().float()
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


def _truth(t, lr, step, b1=0.9, b2=0.999, eps=1e-15):
    p, g, m, v = (t[k].double() for k in "pgmv")
    m1 = m + (1 - b1) * (g - m)
    v1 = b2 * v + (1 - b2) * g * g
    delta = lr / (1 - b1 ** step) * m1 / (v1.sqrt() / math.sqrt(1 - b2 ** step) + eps)
    return p - delta, delta, m1, v1


def _ratios(out, t, truth, rows):
    """max over the edited elements of error / bound for p, m and v."""
    p1, delta, m1, v1 = truth
    sel = rows.view((-1,) + (1,) * (t["p"].dim() - 1)).expand_as(t["p"])
    bound_p = _ulp(p1) + 4 * _ulp(delta)
    r = {}
    for key, got, want, bound in (("p", out[0], p1, bound_p), ("m", out[1], m1, 2 * _ulp(m1)),
                                  ("v", out[2], v1, 2 * _ulp(v1))):
        e = ((got.double() - want).abs() / bound)[sel]
        r[key] = float(e.max()) if e.numel() else 0.0
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("P", [1, 31, 32, 33, 4097, 500_000])
@pytest.mark.parametrize("mask_kind", ["random20", "spatial20", "all", "none", "single"])
def test_one_step_against_fp64_truth(layout, P, mask_kind):
    step0 = 4
    tensors, gen = _inputs(P, LAYOUTS[layout], seed=P * 7 + len(layout))
    pos = torch.randn(P, 3, generator=gen, device="cuda")
    mask = _mask(mask_kind, P, pos, gen)
    # ours on inputs whose unedited g, m, v rows hold NaN: the kernel must neither read nor write them
    poisoned = []
    for t in tensors:
        sel = (~mask).view((-1,) + (1,) * (t["p"].dim() - 1)).expand_as(t["p"])
        poisoned.append(dict(t, **{k: t[k].masked_fill(sel, math.nan) for k in "gmv"}))
    opt, params = _make("masked", poisoned, step0, mask=mask)
    opt.step()
    worst_torch = {}
    results = {}
    for kind in ("foreach", "fused"):
        o, ps = _make(kind, tensors, step0)
        o.step()
        results[kind] = [(q.detach(), o.state[q]["exp_avg"], o.state[q]["exp_avg_sq"]) for q in ps]
    for i, (t, q) in enumerate(zip(tensors, params)):
        st = opt.state[q]
        assert float(st["step"]) == step0 + 1 and st["step"].device.type == "cpu"
        got = (q.detach(), st["exp_avg"], st["exp_avg_sq"])
        un = (~mask).view((-1,) + (1,) * (t["p"].dim() - 1)).expand_as(t["p"])
        for x, before in zip(got, (t["p"], poisoned[i]["m"], poisoned[i]["v"])):
            assert torch.equal(_bits(x)[un], _bits(before)[un]), (t["name"], "unedited row changed")
        assert torch.equal(_bits(q.grad), _bits(poisoned[i]["g"]))
        if not mask.any() or t["p"].numel() == 0:
            continue
        truth = _truth(t, LRS[t["name"]], step0 + 1)
        ours = _ratios(got, t, truth, mask)
        for kind in ("foreach", "fused"):
            for key, r in _ratios(results[kind][i], t, truth, mask).items():
                worst_torch[key] = max(worst_torch.get(key, 0.0), r)
        for key, r in ours.items():
            # the bound is 1 (1 ulp(p) + 4 ulp(update), 2 ulp for m and v); where torch's own Adam misses it on these
            # inputs (a moment that nearly cancels, m + (1 - beta1)(g - m) ~ 0, loses its relative accuracy in any fp32
            # evaluation), the bound is torch's worst case
            assert r <= max(1.0, worst_torch.get(key, 0.0)), (t["name"], key, r, worst_torch)


@pytest.mark.gpu
def test_lr_change_and_steps_of_groups_without_grad():
    P = 4097
    tensors, gen = _inputs(P, SHAPES, seed=3)
    mask = torch.ones(P, dtype=torch.bool, device="cuda")
    ours, po = _make("masked", tensors, 0, mask=mask)
    ref, pr = _make("foreach", tensors, 0)
    for opt in (ours, ref):
        for p in opt.state:
            opt.state[p] = {}   # lazily created at the first step with a gradient, as torch does
    for k in range(4):
        for opt, ps in ((ours, po), (ref, pr)):
            opt.param_groups[0]["lr"] = 1e-3 * (k + 1)
            for i, p in enumerate(ps):
                p.grad = None if (i == 2 and k in (1, 2)) or (i == 4 and k == 0) else tensors[i]["g"] * (k + 1)
            opt.step()
    for a, b in zip(po, pr):
        sa, sb = ours.state[a], ref.state[b]
        assert torch.equal(sa["step"], sb["step"]) and sa["step"].device.type == "cpu"
        assert float((a.detach() - b.detach()).norm() / b.detach().norm()) <= 1e-6
    assert [float(ours.state[p]["step"]) for p in po] == [4, 4, 2, 4, 3, 4]
    # the changed lr was used: xyz moved by the lrs 1e-3 .. 4e-3 (an unchanged 1e-3 would move it ~2.5x less)
    moved = float((po[0].detach() - tensors[0]["p"]).abs().mean())
    assert 5e-3 < moved < 1.5e-2, moved


def _trajectory(kind, tensors, mask, steps=50, drop=None, seed=11):
    """`steps` steps under the edit invariant (zero gradients and moments outside the mask) with a per-step xyz lr
    schedule. `drop` = (step, row): from that step on, the row is left out of the mask."""
    t0 = [dict(t, m=t["m"] * 0, v=t["v"] * 0) for t in tensors]
    opt, params = _make(kind, t0, 0, mask=mask.clone() if kind == "masked" else None)
    for p in opt.state:
        opt.state[p] = {}
    gen = torch.Generator(device="cuda").manual_seed(seed)
    snap = None
    for k in range(steps):
        if drop is not None and k == drop[0]:
            m2 = mask.clone()
            m2[drop[1]] = False
            opt.set_mask(m2)
            snap = [p.detach()[drop[1]].clone() for p in params]
        opt.param_groups[0]["lr"] = 1.6e-4 * 0.01 ** (k / steps)
        for p in params:
            g = torch.randn(p.shape, generator=gen, device="cuda") * 1e-2
            p.grad = torch.where(mask.view((-1,) + (1,) * (p.dim() - 1)), g, 0.0)   # +0.0, as grad_mask writes
        opt.step()
    return opt, params, snap


@pytest.mark.gpu
def test_trajectory_under_the_edit_invariant():
    P = 100_003
    tensors, gen = _inputs(P, SHAPES, seed=5)
    mask = _mask("spatial20", P, tensors[0]["p"], gen)
    res = {k: _trajectory(k, tensors, mask) for k in ("foreach", "fused", "masked")}
    again = _trajectory("masked", tensors, mask)
    for i, t in enumerate(tensors):
        un = (~mask).view((-1,) + (1,) * (t["p"].dim() - 1)).expand_as(t["p"])
        ed = ~un
        get = lambda k: (res[k][1][i].detach(), res[k][0].state[res[k][1][i]]["exp_avg"],
                         res[k][0].state[res[k][1][i]]["exp_avg_sq"])
        ours, fe, fu = get("masked"), get("foreach"), get("fused")
        for x, y, z in zip(ours, fe, fu):
            assert torch.equal(_bits(x)[un], _bits(y)[un]), t["name"]
            rel = lambda a, b: float((a[ed].double() - b[ed].double()).norm() / b[ed].double().norm())
            assert rel(x, y) <= 2 * rel(z, y) + 1e-7, (t["name"], rel(x, y), rel(z, y))
        assert torch.equal(_bits(ours[0])[un], _bits(t["p"])[un])
        rep = again[1][i].detach()
        assert torch.equal(_bits(rep), _bits(ours[0])), "two identical runs differ"
    row = int(torch.nonzero(mask)[0])
    opt, params, snap = _trajectory("masked", tensors, mask, drop=(20, row))
    for p, s in zip(params, snap):
        assert torch.equal(_bits(p.detach()[row]), _bits(s))
    assert not torch.equal(params[0].detach()[row], tensors[0]["p"][row])   # it had moved before it was dropped


@pytest.mark.gpu
def test_capturable_step_replays_in_a_cuda_graph():
    P = 33_333
    tensors, gen = _inputs(P, SHAPES, seed=9)
    mask = _mask("random20", P, None, gen)
    eager, pe = _make("masked", tensors, 2, mask=mask, capturable=True)
    graphed, pg = _make("masked", tensors, 2, mask=mask, capturable=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(3):
            eager.step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.step()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    for a, b in zip(pe, pg):
        sa, sb = eager.state[a], graphed.state[b]
        assert sa["step"].is_cuda and float(sa["step"]) == 5.0
        for key in ("step", "exp_avg", "exp_avg_sq"):
            assert torch.equal(_bits(sa[key]), _bits(sb[key])), key
        assert torch.equal(_bits(a.detach()), _bits(b.detach()))
    assert not torch.equal(pe[0].detach(), tensors[0]["p"])


@pytest.mark.gpu
def test_step_checks_rows_and_devices():
    tensors, gen = _inputs(100, SHAPES, seed=1)
    opt, params = _make("masked", tensors, 0, mask=torch.ones(99, dtype=torch.bool, device="cuda"))
    with pytest.raises(ValueError, match="set_mask"):
        opt.step()
    bad = MaskedAdam([torch.nn.Parameter(torch.zeros(100, 3))], mask=torch.ones(100, dtype=torch.bool, device="cuda"))
    bad.param_groups[0]["params"][0].grad = torch.zeros(100, 3)
    with pytest.raises(ValueError, match="CUDA"):
        bad.step()
    u8 = torch.ones(100, dtype=torch.uint8, device="cuda")
    opt.set_mask(u8)
    assert opt.mask.data_ptr() == u8.data_ptr()
    b = torch.ones(100, dtype=torch.bool, device="cuda")
    opt.set_mask(b)
    assert opt.mask.dtype == torch.uint8 and opt.mask.data_ptr() == b.data_ptr()   # viewed, not copied


def _loop(optimizer, cuda_graph):
    from gaussianeditor_b200.edit_loop import run_edit_loop
    from gaussianeditor_b200.rasterizer import GaussianRasterizer
    return run_edit_loop(functools.partial(GaussianRasterizer, deterministic=True), steps=200, P=200_000,
                         densification_interval=100, deterministic=True, grad_mask="kernel", optimizer=optimizer,
                         cuda_graph=cuda_graph)


def _compare_arms(a, b):
    assert a["counts"] == b["counts"] and len(set(a["counts"])) > 1   # a densification
    assert torch.equal(a["mask"], b["mask"])
    un = ~a["mask"]
    for n, p in a["params"].items():
        assert torch.equal(_bits(p[un]), _bits(b["params"][n][un])), n
    assert max(abs(x - y) for x, y in zip(a["losses"], b["losses"])) <= 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("cuda_graph", [False, True])
def test_edit_loop_masked_optimizer(cuda_graph):
    a = _loop("adam", cuda_graph)
    b = _loop("masked", cuda_graph)
    assert isinstance(b["optimizer"], MaskedAdam) and isinstance(a["optimizer"], torch.optim.Adam)
    assert b["optimizer"].mask.data_ptr() == b["mask"].data_ptr()
    _compare_arms(a, b)


def test_edit_loops_reject_masked_optimizer_without_a_mask():
    from gaussianeditor_b200.edit_loop import run_edit_loop, run_sharded_edit_loop
    with pytest.raises(ValueError, match="grad_mask"):
        run_edit_loop(None, steps=1, P=100, optimizer="masked")
    with pytest.raises(ValueError, match="optimizer"):
        run_edit_loop(None, steps=1, P=100, optimizer="sgd")
    with pytest.raises(ValueError, match="grad_mask"):
        run_sharded_edit_loop(steps=1, P=100, optimizer="masked")


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
def test_world1_sharded_edit_loop_masked_optimizer(nccl_world1):
    from gaussianeditor_b200.edit_loop import run_sharded_edit_loop
    kw = dict(steps=200, P=60000, densification_interval=100, seed=0, mode="dense", deterministic=True,
              grad_mask="kernel")
    a = run_sharded_edit_loop(optimizer="adam", **kw)
    b = run_sharded_edit_loop(optimizer="masked", **kw)
    assert len(a["densify"]) == 1
    assert b["optimizer"].mask.data_ptr() == b["mask"].data_ptr()   # re-set to the mask rebalance carried
    _compare_arms(a, b)
