"""Tiny end-to-end scenario for compute-sanitizer (memcheck / racecheck): every kernel family on a small cloud.

    compute-sanitizer --tool memcheck python tools/sanitize_case.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gaussianeditor_b200 import _lib, sharded as S, synth  # noqa: E402
from gaussianeditor_b200.rasterizer import GaussianRasterizer  # noqa: E402
from util import cloud_tensors, run_ours, settings_from  # noqa: E402

dev = torch.device("cuda")
cloud, _ = synth.make_config("c3", P=3001)
cam = synth.ring_cameras(8, 4.5, 15.0, 200, 136, 61.0)[2]   # partial last tile column and row
dL = np.random.default_rng(0).uniform(size=(3, cam.image_height, cam.image_width)).astype(np.float32)

for fv in (0, 1, 2, 3, 4, 5):
    _lib.set_option("render_fwd_variant", fv)
    run_ours(cloud, cam, (0.1, 0.2, 0.3))
_lib.set_option("render_fwd_variant", 3)
for bv in (0, 1, 2, 3, 4, 6, 7, 8):
    _lib.set_option("render_bwd_variant", bv)
    run_ours(cloud, cam, (0.1, 0.2, 0.3), dL=dL)
_lib.set_option("render_bwd_variant", 4)
run_ours(cloud, cam, (0, 0, 0), dL=dL, colors_precomp=np.random.default_rng(1).random((3001, 3), dtype=np.float32))
for M, deg in ((9, 2), (4, 1), (1, 0)):                      # non-TMA SH paths
    c2 = synth.Cloud(means3D=cloud.means3D, scales=cloud.scales, rotations=cloud.rotations, opacities=cloud.opacities,
                     shs=np.ascontiguousarray(cloud.shs[:, :M]), sh_degree=deg)
    run_ours(c2, cam, (0, 0, 0), dL=dL)

# semantic tracing + markVisible
rs = settings_from(cam, (0, 0, 0), cloud.sh_degree, dev)
rast = GaussianRasterizer(rs)
ct = cloud_tensors(cloud, dev)
w = torch.zeros(3001, 1, device=dev); cnt = torch.zeros(3001, 1, dtype=torch.int32, device=dev)
rast.apply_weights(ct["means3D"], torch.zeros_like(ct["means3D"]), ct["opacities"], None, w, ct["scales"], ct["rotations"], None,
                   cnt, (torch.rand(1, cam.image_height, cam.image_width, device=dev) > 0.5).float())
rast.markVisible(ct["means3D"])

# fused activations (bulk block path needs P % 4 == 0 rows in the last block: run both)
for P in (3001, 3072):
    cl, _ = synth.make_config("c3", P=P)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    op = t(cl.opacities).clamp(1e-6, 1 - 1e-6)
    raw = [t(cl.means3D), torch.zeros(P, 3, device=dev), torch.log(op / (1 - op)), t(cl.shs[:, :1]).contiguous(),
           t(cl.shs[:, 1:]).contiguous(), torch.log(t(cl.scales)), t(cl.rotations) * 2.0]
    raw = [x.requires_grad_(True) for x in raw]
    col, _, _ = rast.forward_raw(*raw)
    (col * torch.from_numpy(dL).to(dev)).sum().backward()

# Gaussian-sharded path, two virtual ranks on this GPU
empty = torch.empty(0, device=dev)
plans = [S.ShardPlan(3001, 2, r) for r in range(2)]
geom = radii = None
bufs = []
for p in plans:
    sl = lambda x: S.shard_slice(x, p)
    b = S.shard_preprocess(p, rs, sl(ct["means3D"]), sl(ct["shs"]), empty, sl(ct["opacities"]), sl(ct["scales"]),
                           sl(ct["rotations"]), empty, geom=geom, radii=radii)
    geom, radii = b.geom, b.radii
    bufs.append(b)
for b in bufs:   # the ranks run one after the other on the shared arrays (no clone: keeps initcheck quiet)
    S.shard_order(b)
    frame = torch.zeros(4, cam.image_height, cam.image_width, device=dev)
    S.shard_render(b, frame[:3], frame[3:])
    acc = S.shard_backward_render(b, torch.from_numpy(dL).to(dev))
    S.shard_backward_preprocess(b, acc[b.plan.base:b.plan.base + b.plan.slice_len].contiguous())

# round 2: both binning implementations x both depth orders, a speculative overflow (second half redone), the alpha
# image with gradient, the camera gradients
import gaussianeditor_b200.rasterizer as RZ
for bvar, dvar in ((0, 0), (1, 1), (1, 0)):
    _lib.set_option("binning_variant", bvar)
    _lib.set_option("depth_sort_variant", dvar)
    run_ours(cloud, cam, (0.1, 0.2, 0.3), dL=dL)
    RZ._r_hint[(0, 3001, cam.image_width, cam.image_height)] = 10      # hopeless guess: overflow path
    run_ours(cloud, cam, (0.1, 0.2, 0.3), dL=dL)
_lib.set_option("binning_variant", 1)
_lib.set_option("depth_sort_variant", 0)
view = rs.viewmatrix.clone().requires_grad_(True)
rs_cam = rs._replace(viewmatrix=view, projmatrix=rs.projmatrix.clone().requires_grad_(True),
                     campos=rs.campos.clone().requires_grad_(True))
# camera gradients + alpha output. initcheck does not track TMA bulk stores (cp.async.bulk shared->global) as writes, so a
# cudaMemcpy of the dL/dSH tensor they fill (autograd's copy into .grad) is reported as "uninitialized" byte for byte
# (one report per 32 bytes of the tensor). The TMA variant therefore runs with SH detached
# (kernel identical, autograd drops the tensor without a copy) and the plain-store variant runs with SH attached.
for pv, sh_grad in ((1, False), (0, True)):
    _lib.set_option("preprocess_variant", pv)
    ctg = cloud_tensors(cloud, dev, requires_grad=True)
    shs = ctg["shs"] if sh_grad else ctg["shs"].detach()
    out = GaussianRasterizer(rs_cam, return_alpha=True, camera_grad=True)(
        means3D=ctg["means3D"], means2D=torch.zeros_like(ctg["means3D"]), opacities=ctg["opacities"], shs=shs,
        scales=ctg["scales"], rotations=ctg["rotations"])
    ((out[0] * torch.from_numpy(dL).to(dev)).sum() + out[3].sum()).backward()
_lib.set_option("preprocess_variant", 1)

# sparse exchange, three virtual ranks on this GPU (tight capacity)
from gaussianeditor_b200 import sparse_sharded as SS
splans = [S.ShardPlan(3001, 3, r) for r in range(3)]
ranks = [SS.SparseRank(p, dev, cam.image_width, cam.image_height) for p in splans]
SS.link_virtual(ranks)


def sparse_forward(cap):
    for rk in ranks:
        rk.matrix.zero_()
    steps = []
    for rk in ranks:
        sl = lambda x: S.shard_slice(x, rk.plan)
        steps.append(SS.sparse_preprocess(rk, rs, sl(ct["means3D"]), sl(ct["shs"]), empty, sl(ct["opacities"]),
                                          sl(ct["scales"]), sl(ct["rotations"]), empty, cap))
    m = torch.stack([rk.matrix for rk in ranks]).sum(0)
    for rk in ranks:
        rk.matrix.copy_(m)
    return steps, [SS.sparse_order(st) for st in steps]


steps, res = sparse_forward(ranks[0].cap_alloc)
steps, res = sparse_forward(max(res[0][1], 1))
for rk in ranks:
    rk.frame.zero_()
for st in steps:
    SS.sparse_render(st, st.rk.frame[:3], st.rk.frame[3:])
for rk in ranks:
    SS.frame_broadcast(rk)
accs = [SS.sparse_backward_render(st, torch.from_numpy(dL).to(dev)) for st in steps]
for st, a in zip(steps, accs):
    SS.sparse_return(st, a)
for st in steps:
    SS.sparse_backward_preprocess(st)
torch.cuda.synchronize()
print("SANITIZE_CASE_DONE")
