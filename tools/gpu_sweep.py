"""Timing sweep over the library's kernel variants on config 3 (per-stage CUDA-event times, ms, median of 5 repeats of
12 steps each after 4 warm-up steps). Every option is swept with the others at their defaults; prints one JSON line.

    python tools/gpu_sweep.py
"""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from gaussianeditor_b200 import _lib  # noqa: E402

SWEEP = {"render_fwd_variant": ([0, 1, 2, 3, 4, 5], ["render_fwd"]),
         "render_bwd_variant": (list(range(15)), ["render_bwd"]),
         "preprocess_variant": ([0, 1], ["preprocess_fwd", "preprocess_bwd"]),
         "binning_variant": ([0, 1], ["emit_instances", "tile_sort", "tile_ranges"]),
         "depth_sort_variant": ([0, 1], ["depth_order_scan"])}

wl = bench.Workload("c3", torch.device("cuda", 0))
r = bench.OursRunner(wl)


def stage_times(n=12, repeats=5):
    for i in range(4):
        r.step(i)
    runs = []
    for _ in range(repeats):
        _lib.set_option("profile", 1)
        _lib.profile_read()
        for i in range(n):
            r.step(i)
        p = _lib.profile_read()
        _lib.set_option("profile", 0)
        runs.append({k: v[0] / max(v[1], 1) for k, v in p.items() if v[1]})
    return {k: round(statistics.median(x[k] for x in runs), 4) for k in runs[0]}


res = {"device": torch.cuda.get_device_name(0), "default": stage_times()}
for opt, (values, stages) in SWEEP.items():
    default = _lib.load().gsr_get_option(opt.encode())
    for v in values:
        _lib.set_option(opt, v)
        t = stage_times()
        res[f"{opt}={v}"] = {s: t.get(s) for s in stages}
    _lib.set_option(opt, default)
print(json.dumps(res))
