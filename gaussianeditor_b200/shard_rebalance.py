"""Densify / prune of a Gaussian-sharded cloud (DESIGN.md 7.2, "Rebalancing").

GaussianEditor clones and prunes Gaussians every ``densification_interval`` steps, so the cloud changes size. A sharded
cloud is laid out by ``ShardPlan(P_total, world, rank)``: rank g holds the rows ``[g*L, g*L + n_g)``. After each rank
has densified and pruned its own rows (``optim_surgery``), the rows are moved so that the cloud is laid out by
``ShardPlan(P_new, world, rank)`` again, in the global order a single-GPU ``densification_postfix`` would give:

  * every rank describes its new local rows as K segments (e.g. K = 2: kept rows, then clones; K = 3: kept rows, split
    copy 1, split copy 2), each in local index order;
  * the new global order is segment-major, rank-minor: (r=0,k=0) (r=1,k=0) ... (r=G-1,k=0) (r=0,k=1) ... With K = 2 the
    kept rows stay in index order and the appended rows follow in index order, as ``cat((kept, clones))`` on one GPU;
    with K = 3 it is ``repeat(2, 1)`` of the split rows after the kept rows;
  * ``rebalance_plan`` turns the all-gathered [world, K] count matrix into the new plans, the (source, destination)
    split sizes and, per destination, the pieces that put the rows it receives (grouped by source rank by the
    all-to-all) back in (segment, rank) order. It depends only on the count matrix, so every rank computes the same;
  * ``rebalance`` packs every parameter row, its row-aligned optimizer state (Adam's ``exp_avg`` / ``exp_avg_sq``) and
    every extra per-Gaussian tensor as bytes into one [n, row_bytes] buffer and moves it with ONE
    ``all_to_all_single``: rows arrive bit-identical to what their source held.

``global_top_k`` selects the same global set of Gaussians on every rank (the densification candidates).
"""
from __future__ import annotations

import math
import zlib
from typing import List, NamedTuple, Optional, Sequence

import torch
import torch.nn as nn

from .sharded import Exchange, ShardPlan

MAX_SEGMENTS = 8   # segments per rebalance (the header all-gather has a fixed size, so that no rank can hang on it)


class Piece(NamedTuple):
    """A run of rows one destination receives: ``length`` rows of segment ``seg`` from rank ``src``, found at
    ``src_off`` in the chunk ``src`` sends to this destination, going to ``dst_off`` in the destination's new slice."""
    src: int
    seg: int
    src_off: int
    length: int
    dst_off: int


class RebalancePlan(NamedTuple):
    """``plans[d]``: the new ShardPlan of rank d. ``splits[r][d]``: rows rank r sends to rank d (send split sizes of r
    are ``splits[r]``, receive split sizes of d are ``[splits[r][d] for r]``). ``pieces[d]``: destination d's pieces,
    ordered by ``dst_off``. ``sends[r]``: rank r's runs ``(dest, seg, local offset, length)`` in send order
    (destination, segment, local order)."""
    plans: List[ShardPlan]
    splits: List[List[int]]
    pieces: List[List[Piece]]
    sends: List[List[tuple]]

    def send_index(self, rank: int, device=None) -> torch.Tensor:
        """Local row indices of `rank` in the order it packs them (int64)."""
        parts = [torch.arange(off, off + n, dtype=torch.int64) for _, _, off, n in self.sends[rank]]
        idx = torch.cat(parts) if parts else torch.empty(0, dtype=torch.int64)
        return idx.to(device) if device is not None else idx

    def recv_index(self, rank: int, device=None) -> torch.Tensor:
        """For each row of `rank`'s new slice, its row in the receive buffer (chunks in source-rank order)."""
        world = len(self.plans)
        base = [sum(self.splits[q][rank] for q in range(r)) for r in range(world)]
        idx = torch.empty(self.plans[rank].count, dtype=torch.int64)
        for pc in self.pieces[rank]:
            s = base[pc.src] + pc.src_off
            idx[pc.dst_off:pc.dst_off + pc.length] = torch.arange(s, s + pc.length, dtype=torch.int64)
        return idx.to(device) if device is not None else idx


def rebalance_plan(counts, world: int) -> RebalancePlan:
    """The new layout of a cloud whose rank r now holds ``counts[r, k]`` rows in segment k (int [world, K]); see the
    module docstring for the order. Raises ValueError for a malformed matrix and when the new cloud would be empty."""
    c = torch.as_tensor(counts, dtype=torch.int64).cpu()
    if c.dim() != 2 or c.size(0) != world or c.size(1) < 1:
        raise ValueError(f"counts must be an int matrix [world={world}, K>=1], got shape {tuple(c.shape)}")
    if bool((c < 0).any()):
        raise ValueError("segment counts must be >= 0")
    c = c.tolist()
    K = len(c[0])
    P_new = sum(sum(row) for row in c)
    if P_new == 0:
        raise ValueError("rebalance would leave an empty cloud (0 Gaussians on every rank)")
    plans = [ShardPlan(P_new, world, d) for d in range(world)]
    start, pos = {}, 0                       # global start of block (r, k): segment-major, rank-minor
    for k in range(K):
        for r in range(world):
            start[r, k] = pos
            pos += c[r][k]
    splits = [[0] * world for _ in range(world)]
    sends = [[] for _ in range(world)]
    pieces = [[] for _ in range(world)]
    for r in range(world):
        local = 0
        seg_local = []
        for k in range(K):
            seg_local.append(local)
            local += c[r][k]
        for d in range(world):
            lo_d, hi_d = plans[d].base, plans[d].base + plans[d].count
            for k in range(K):
                s, e = start[r, k], start[r, k] + c[r][k]
                lo, hi = max(s, lo_d), min(e, hi_d)
                if hi <= lo:
                    continue
                n = hi - lo
                sends[r].append((d, k, seg_local[k] + lo - s, n))
                pieces[d].append(Piece(r, k, splits[r][d], n, lo - lo_d))
                splits[r][d] += n
    for p in pieces:
        p.sort(key=lambda pc: pc.dst_off)
    return RebalancePlan(plans, splits, pieces, sends)


# ---------------------------------------------------------------------------------------------------------
# rows as bytes
# ---------------------------------------------------------------------------------------------------------
def row_spec(t: torch.Tensor) -> tuple:
    """(dtype, row shape, bytes per row) of a per-Gaussian tensor."""
    row = tuple(t.shape[1:])
    return t.dtype, row, int(math.prod(row)) * t.element_size()


def pack_rows(tensors: Sequence[torch.Tensor], index: torch.Tensor) -> torch.Tensor:
    """Rows `index` of every tensor (same first dimension), as bytes side by side: uint8 [len(index), row_bytes]."""
    cols = []
    for t in tensors:
        _, row, nb = row_spec(t)
        if nb == 0:
            continue
        n = t.shape[0]
        b = t.detach().contiguous().reshape(n, int(math.prod(row))).view(torch.uint8)
        cols.append(b.index_select(0, index))
    if not cols:
        return torch.empty(index.numel(), 0, dtype=torch.uint8, device=index.device)
    return torch.cat(cols, dim=1)


def unpack_rows(buf: torch.Tensor, specs: Sequence[tuple]) -> List[torch.Tensor]:
    """Inverse of pack_rows: the tensors of `specs` ((dtype, row shape, bytes per row) each) from buf [n, row_bytes]."""
    n = buf.shape[0]
    out, o = [], 0
    for dtype, row, nb in specs:
        if nb == 0:
            out.append(torch.empty((n,) + tuple(row), dtype=dtype, device=buf.device))
            continue
        out.append(buf[:, o:o + nb].contiguous().view(dtype).reshape((n,) + tuple(row)))
        o += nb
    return out


def _row_aligned_state(optimizer, p: torch.Tensor) -> list:
    """The state keys of `p` that move with its rows (optim_surgery._swap's rule), in a fixed order."""
    state = optimizer.state.get(p)
    if not state:
        return []
    return sorted(k for k, v in state.items() if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == p.shape[0])


# ---------------------------------------------------------------------------------------------------------
# the collectives
# ---------------------------------------------------------------------------------------------------------
_REASONS = {1: "segment counts negative or more than %d segments" % MAX_SEGMENTS,
            2: "a tensor's first dimension is not the sum of the rank's segment counts",
            3: "a param group does not hold exactly one tensor",
            4: "tensors on a device the process group's backend cannot exchange (NCCL: one CUDA device, gloo: CPU)",
            5: "the plan does not match the process group (world / rank)"}


def _header_device(exchange: Exchange):
    if exchange.backend == "nccl":
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def rebalance(exchange: Exchange, plan: ShardPlan, segment_counts: Sequence[int], optimizer=None,
              extras: Sequence[torch.Tensor] = (), stats: Optional[dict] = None):
    """Move this rank's rows to their owners under the new cloud size (collective: every rank calls it once).

    `segment_counts`: the K sizes of this rank's local segments (rows of every tensor, in local order). `optimizer`:
    every param group holds one row-aligned tensor (optim_surgery's contract); parameters and their row-aligned state
    tensors move, scalar state (``step``, also capturable Adam's device ``step``) is untouched, and new ``nn.Parameter``s
    are swapped into the groups. `extras`: any other per-Gaussian tensors (a bool mask, an int64 generation, ...).

    Malformed input on any rank (a first dimension that is not the sum of the segments, a different set of tensors on
    different ranks, an empty new cloud) raises the same ValueError on every rank after one small all-gather, before any
    row moves. `stats` (a dict, optional) receives ``row_bytes``, ``rows_moved`` and ``bytes_moved`` (rows that change
    rank, over the whole group). Returns ``(new plan of this rank, moved extras)``."""
    world, rank = exchange.world, exchange.rank
    counts = [int(x) for x in segment_counts]
    K = len(counts)
    n = sum(counts)
    code = 0
    if K < 1 or K > MAX_SEGMENTS or any(x < 0 for x in counts):
        code = 1
    if plan.world != world or plan.rank != rank:
        code = code or 5
    groups = list(optimizer.param_groups) if optimizer is not None else []
    moved, specs, layout, where = [], [], [], []    # where: ("param", group) / ("state", group, key) / ("extra", i)
    for gi, group in enumerate(groups):
        if len(group["params"]) != 1:
            code = code or 3
            continue
        p = group["params"][0]
        for key in ["<param>"] + _row_aligned_state(optimizer, p):
            t = p if key == "<param>" else optimizer.state[p][key]
            moved.append(t)
            where.append(("param", gi) if key == "<param>" else ("state", gi, key))
            layout.append(f"{gi}/{group.get('name', '')}/{key}")
    for i, t in enumerate(extras):
        moved.append(t)
        where.append(("extra", i))
        layout.append(f"extra{i}")
    for t in moved:
        specs.append(row_spec(t))
        if t.dim() == 0 or t.shape[0] != n:
            code = code or 2
    devices = {t.device for t in moved}
    if len(devices) > 1 or any((d.type == "cuda") != (exchange.backend == "nccl") for d in devices):
        code = code or 4
    crc = zlib.crc32("|".join(f"{tag}:{s[0]}:{s[1]}" for tag, s in zip(layout, specs)).encode())
    # one small all-gather: [code, layout crc, K, counts padded to MAX_SEGMENTS]
    hw = 3 + MAX_SEGMENTS
    head = torch.zeros(world * hw, dtype=torch.int64, device=_header_device(exchange))
    mine = [code, crc, K] + (counts + [0] * MAX_SEGMENTS)[:MAX_SEGMENTS]
    if code == 1:
        mine[3:] = [0] * MAX_SEGMENTS
    head[rank * hw:(rank + 1) * hw] = torch.tensor(mine, dtype=torch.int64)
    exchange.all_gather_inplace(head)
    head = head.view(world, hw).cpu().tolist()
    bad = [(r, h[0]) for r, h in enumerate(head) if h[0] != 0]
    if bad:
        raise ValueError("rebalance: malformed input on " + "; ".join(f"rank {r}: {_REASONS[c]}" for r, c in bad))
    if len({h[2] for h in head}) != 1:
        raise ValueError(f"rebalance: the ranks passed different numbers of segments {[h[2] for h in head]}")
    if len({h[1] for h in head}) != 1:
        raise ValueError("rebalance: the ranks move different sets of tensors (param groups, optimizer state or "
                         "extras differ in number, names, dtype or row shape)")
    matrix = [h[3:3 + K] for h in head]
    rb = rebalance_plan(matrix, world)      # raises the same ValueError on every rank for an empty cloud
    new_plan = rb.plans[rank]
    row_bytes = sum(s[2] for s in specs)
    if stats is not None:
        rows = sum(rb.splits[r][d] for r in range(world) for d in range(world) if r != d)
        stats.update(row_bytes=row_bytes, rows_moved=rows, bytes_moved=rows * row_bytes)
    if not moved:
        return new_plan, []
    device = next(iter(devices))
    send = pack_rows(moved, rb.send_index(rank, device))
    recv = torch.empty(sum(rb.splits[r][rank] for r in range(world)), row_bytes, dtype=torch.uint8, device=device)
    if row_bytes > 0:
        exchange.all_to_all_single(recv, send, [rb.splits[r][rank] for r in range(world)], rb.splits[rank])
    new = unpack_rows(recv.index_select(0, rb.recv_index(rank, device)), specs)
    out_extras = []
    new_params = {}
    for w, t in zip(where, new):
        if w[0] == "param":
            new_params[w[1]] = t
        elif w[0] == "extra":
            out_extras.append(t)
    for gi, group in enumerate(groups):   # swap the parameters, then the state that follows their rows
        old = group["params"][0]
        state = optimizer.state.pop(old, None)
        p = nn.Parameter(new_params[gi], requires_grad=old.requires_grad)
        group["params"][0] = p
        if state is not None:
            for w, t in zip(where, new):
                if w[0] == "state" and w[1] == gi:
                    state[w[2]] = t
            optimizer.state[p] = state
    return new_plan, out_extras


def kth_pair(values: torch.Tensor, k: int):
    """(value, index) of the k-th largest entry of `values` [n] under the order (value descending, index ascending), as
    two python numbers (value exact: a float32 is exact in a double). NaN counts as 0."""
    v = torch.nan_to_num(values.detach().reshape(-1), nan=0.0, posinf=float("inf"), neginf=float("-inf"))
    order = torch.sort(v, descending=True, stable=True).indices
    i = int(order[k - 1])
    return float(v[i]), i


def select_against(values: torch.Tensor, base: int, pair) -> torch.Tensor:
    """Rows of `values` (global indices base, base+1, ...) that come before or at `pair` in that order: bool [n]."""
    v = torch.nan_to_num(values.detach().reshape(-1), nan=0.0, posinf=float("inf"), neginf=float("-inf"))
    thr = torch.tensor(pair[0], dtype=v.dtype, device=v.device)
    gidx = base + torch.arange(v.numel(), device=v.device)
    return (v > thr) | ((v == thr) & (gidx <= pair[1]))


def top_k_mask(values: torch.Tensor, k: int) -> torch.Tensor:
    """The single-process rule global_top_k reproduces: exactly k rows, ties broken by the lower index."""
    return select_against(values, 0, kth_pair(values, k))


def global_top_k(exchange: Exchange, plan: ShardPlan, local_values: torch.Tensor, k: int) -> torch.Tensor:
    """Collective: this rank's rows (bool [plan.count]) of the k largest values of the whole cloud, ties broken by the
    lower global index, so exactly k rows are selected over all ranks and every rank agrees. One all-gather of the
    values into [P_pad] (padding -inf, NaN counts as 0), rank 0 finds the k-th (value, index) pair and broadcasts it.
    A malformed input (`local_values` not [plan.count], k outside [1, P_total]) raises ValueError on every rank."""
    v = local_values.detach().reshape(-1)
    ok = v.numel() == plan.count and 1 <= int(k) <= plan.P_total and plan.world == exchange.world
    L = plan.slice_len
    dev = _header_device(exchange)
    total = torch.full((exchange.world, L + 1), float("-inf"), dtype=torch.float32, device=dev)
    if ok:
        total[exchange.rank, :plan.count] = torch.nan_to_num(v.float(), nan=0.0, posinf=float("inf"),
                                                             neginf=float("-inf")).to(dev)
    total[exchange.rank, L] = 0.0 if ok else 1.0
    exchange.all_gather_inplace(total)
    if bool((total[:, L] != 0).any()):
        bad = [r for r in range(exchange.world) if float(total[r, L]) != 0]
        raise ValueError(f"global_top_k: malformed input on rank(s) {bad} (values must be the rank's [plan.count] rows "
                         f"and k in [1, P_total])")
    pair = torch.zeros(2, dtype=torch.float64, device=dev)
    if exchange.rank == 0:
        val, idx = kth_pair(total[:, :L].reshape(-1), int(k))
        pair[0], pair[1] = val, idx
    exchange.broadcast(pair, 0)
    pair = pair.cpu().tolist()
    sel = select_against(v.float(), plan.base, (pair[0], int(pair[1])))
    return sel.to(local_values.device)
