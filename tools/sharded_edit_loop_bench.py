"""Config 5 on a Gaussian-sharded cloud, densify and prune included (edit_loop.run_sharded_edit_loop): ms per step and,
per densification, ms of selection, surgery, rebalance and rasterizer re-creation, and the bytes moved across ranks.

    python tools/sharded_edit_loop_bench.py [--steps 200] [--modes dense,sparse]          # world 1
    torchrun --nproc-per-node=N tools/sharded_edit_loop_bench.py ...                       # N GPUs

Prints one JSON line per mode (rank 0), with the card's name and power limit read in the same run. Times are the
largest over the ranks."""
import argparse
import json
import os
import socket
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in q.stdout.strip().split(",")[:2]]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--P", type=int, default=None)
    ap.add_argument("--interval", type=int, default=100)
    ap.add_argument("--modes", default="dense,sparse")
    ap.add_argument("--deterministic", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    if "RANK" not in os.environ:   # one process without torchrun
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from gaussianeditor_b200.distributed import max_over_ranks
    from gaussianeditor_b200.edit_loop import run_sharded_edit_loop
    from gaussianeditor_b200.sharded import init_distributed
    import torch.distributed as dist
    init_distributed("nccl")
    dev = torch.device("cuda", torch.cuda.current_device())
    name, power = card()
    try:
        for mode in a.modes.split(","):
            kw = dict(P=a.P, mode=mode, deterministic=a.deterministic)
            run_sharded_edit_loop(steps=a.interval + 2, densification_interval=a.interval, **kw)   # warm-up
            out = run_sharded_edit_loop(steps=a.steps, densification_interval=a.interval, **kw)
            phases = {}
            for key in ("select", "surgery", "rebalance", "recreate"):
                vals = [max_over_ranks(d[key], dev) for d in out["densify"]]
                phases[key + "_ms"] = [round(v, 3) for v in vals]
            res = dict(world=out["world"], mode=out["mode"], steps=a.steps, interval=a.interval,
                       deterministic=a.deterministic, P_first=out["P_first"], P_last=out["P_last"],
                       ms_per_step=round(max_over_ranks(out["ms_per_step"], dev), 4),
                       densify_bytes_moved=[d["bytes_moved"] for d in out["densify"]],
                       densify_rows_moved=[d["rows_moved"] for d in out["densify"]], **phases, gpu=name,
                       power_limit=power)
            if dist.get_rank() == 0:
                print(json.dumps(res), flush=True)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
