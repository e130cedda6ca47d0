"""A plain numpy model of how the device merge cuts its input into tiles.

Restated from the partition described in DESIGN.md and the merge's level sizing, independently of the CUDA code:

* Levels.  Level 0 is every row a run contributes (rows before the run's start row are skipped).  Level l + 1 holds
  every S-th key of level l: with stride = S**l, run r's level-l samples are the rows
  ``row0[r] + (j + 1) * stride - 1`` for ``j < (n[r] - row0[r]) // stride``.  Levels are added while a level has
  more than PLAN_TILE keys; the last one (``top``) is merged as one tile.
* Splitters.  With ``q = PLAN_TILE // S - 2k``, level l < top is cut into ``ceil(total[l + 1] / q)`` tiles; tile t
  starts at the key ``sorted(level l + 1)[t * q]``.
* Bounds.  Tile t of run r starts at the lower bound of its splitter in run r's level-l keys, in the true key
  order.  All rows of one key therefore fall into one tile.
* Emit tiles.  The output is written by emit tiles of two consecutive plan tiles (level-0 tiles); the last one
  may be single.  An emit tile's first output row is the number of rows all plan tiles before it emit.

Keys are given as per-run arrays of *ordinals*: any numpy values whose order is the key order (the integer key
itself, or a rank from ``key_ranks``).  Sequence numbers and row kinds decide which key groups produce a row.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

S = 16
PLAN_TILE = 2048


def tile_bound(k: int) -> int:
    """Most rows a tile below the top level can hold: S(q + k - 1) + k(S - 1)."""
    q = PLAN_TILE // S - 2 * k
    return S * (q + k - 1) + k * (S - 1)


def true_key(fields: Sequence) -> tuple:
    """Sort key of one primary key in the comparator's order: integers signed, BOOLEAN false < true, strings and
    binaries unsigned bytewise then by length (Python bytes order), field by field."""
    out = []
    for v in fields:
        if isinstance(v, str):
            out.append(v.encode())
        elif isinstance(v, (bytes, bytearray)):
            out.append(bytes(v))
        else:
            out.append(int(v))
    return tuple(out)


def key_ranks(runs_keys: Sequence[Sequence[Sequence]]) -> List[np.ndarray]:
    """Per-run key tuples -> per-run int64 ranks in the true key order (equal keys, equal rank)."""
    uniq = sorted({true_key(kt) for keys in runs_keys for kt in keys})
    rank = {kt: i for i, kt in enumerate(uniq)}
    return [np.array([rank[true_key(kt)] for kt in keys], np.int64) for keys in runs_keys]


# ---- which key groups emit a row (members in sequence order, oldest first)
RETRACT = (1, 3)          # UPDATE_BEFORE, DELETE
# "all":           every key group (deduplicate, partial-update, aggregate without drop-delete)
# "drop_delete":   the result takes the newest member's kind and retract results are dropped (deduplicate, or
#                  partial-update with remove-record-on-delete over INSERT / DELETE rows, under drop-delete)
# "ignore_delete": retract members are skipped, so a group of retracts only is empty (deduplicate / first-row)
RULES = ("all", "drop_delete", "ignore_delete")


@dataclass
class TilePlan:
    k: int                              # runs that take part (with rows)
    q: int
    level_total: List[int]
    n_tiles_per_level: List[int]
    bounds: List[np.ndarray]            # per level below top: [n_tiles + 1, k] level-local bounds
    tile_sizes: List[np.ndarray]        # per level below top: rows per tile
    bounds0: np.ndarray                 # level 0, absolute rows: [n_tiles + 1, k]
    order_run: np.ndarray = field(default=None)
    order_row: np.ndarray = field(default=None)
    plan_rows: Optional[np.ndarray] = None     # output rows per plan tile
    plan_bytes: Optional[np.ndarray] = None    # output payload bytes per plan tile (one var-len column)

    @property
    def n_levels(self) -> int:
        """Levels above level 0 (what the merge statistics call n_levels)."""
        return len(self.level_total) - 1

    @property
    def n_tiles(self) -> int:
        return self.n_tiles_per_level[0]

    @property
    def largest_tile(self) -> int:
        """Largest tile of any level below the top one (the top level is one tile of <= PLAN_TILE keys)."""
        return max((int(s.max()) for s in self.tile_sizes if len(s)), default=0)

    @property
    def n_emit_tiles(self) -> int:
        return (self.n_tiles + 1) // 2

    def emit_rows(self) -> np.ndarray:
        r = np.append(self.plan_rows, 0) if self.n_tiles % 2 else self.plan_rows
        return r.reshape(-1, 2).sum(axis=1)

    def emit_bytes(self) -> np.ndarray:
        b = np.append(self.plan_bytes, 0) if self.n_tiles % 2 else self.plan_bytes
        return b.reshape(-1, 2).sum(axis=1)

    def out_base(self) -> np.ndarray:
        """First output row of every emit tile."""
        before = np.concatenate([[0], np.cumsum(self.plan_rows)])
        return before[0:self.n_tiles:2]


def plan(ordinals: Sequence[np.ndarray], start_rows: Optional[Sequence[int]] = None,
         seqs: Optional[Sequence[np.ndarray]] = None, kinds: Optional[Sequence[np.ndarray]] = None,
         rule: str = "all", value_lens: Optional[Sequence[np.ndarray]] = None) -> TilePlan:
    """Tile structure of a merge of runs whose keys have the given ordinals (strictly increasing per run).

    With `seqs` and `kinds`, also the merged order (key, then sequence number) and each plan tile's output rows
    under `rule` (see RULES); with `value_lens` too (per run, payload bytes of one var-len value column, 0 for NULL), each plan
    tile's output bytes of a deduplicate merge of that column."""
    k = len(ordinals)
    ords = [np.asarray(o) for o in ordinals]
    n = [len(o) for o in ords]
    row0 = list(start_rows) if start_rows is not None else [0] * k
    # runs without rows (after their start row) do not take part in the merge
    k_live = sum(1 for r in range(k) if n[r] > row0[r])
    q = PLAN_TILE // S - 2 * k_live
    assert q >= 1, "too many runs for one merge"

    def level_keys(lvl: int, r: int) -> np.ndarray:
        stride = S ** lvl
        cnt = (n[r] - row0[r]) // stride
        return ords[r][row0[r] + (np.arange(cnt, dtype=np.int64) + 1) * stride - 1]

    level_total = []
    while True:
        lvl = len(level_total)
        tot = sum((n[r] - row0[r]) // S ** lvl for r in range(k))
        level_total.append(tot)
        if tot <= PLAN_TILE:
            break
    top = len(level_total) - 1
    n_tiles = [0] * (top + 1)
    n_tiles[top] = 1
    for lvl in range(top - 1, -1, -1):
        n_tiles[lvl] = -(-level_total[lvl + 1] // q)

    bounds, sizes = [], []
    for lvl in range(top):
        above = np.sort(np.concatenate([level_keys(lvl + 1, r) for r in range(k)]))
        splitters = above[np.arange(1, n_tiles[lvl], dtype=np.int64) * q]
        b = np.zeros((n_tiles[lvl] + 1, k), np.int64)
        for r in range(k):
            keys = level_keys(lvl, r)
            b[1:-1, r] = np.searchsorted(keys, splitters, side="left")
            b[-1, r] = len(keys)
        bounds.append(b)
        sizes.append(np.diff(b, axis=0).sum(axis=1))
    if top == 0:
        b0 = np.array([[0] * k, [n[r] - row0[r] for r in range(k)]], np.int64)
    else:
        b0 = bounds[0]
    bounds0 = b0 + np.array(row0, np.int64)[None, :]
    tp = TilePlan(k_live, q, level_total, n_tiles, bounds, sizes, bounds0)
    if seqs is None:
        return tp

    # merged order: key, then sequence number (what the LoserTree pops)
    run_id = np.concatenate([np.full(n[r] - row0[r], r, np.int64) for r in range(k)] or [np.zeros(0, np.int64)])
    row_id = np.concatenate([np.arange(row0[r], n[r], dtype=np.int64) for r in range(k)] or [np.zeros(0, np.int64)])
    key = np.concatenate([ords[r][row0[r]:] for r in range(k)]) if k else np.zeros(0)
    seq = np.concatenate([np.asarray(seqs[r])[row0[r]:] for r in range(k)]) if k else np.zeros(0)
    order = np.lexsort((seq, key))
    tp.order_run, tp.order_row = run_id[order], row_id[order]
    if kinds is None:
        return tp
    kind = np.concatenate([np.asarray(kinds[r])[row0[r]:] for r in range(k)])[order]
    # plan tile of every merged row (all rows of a key share one)
    tile_of = np.empty(len(order), np.int64)
    for r in range(k):
        m = tp.order_run == r
        tile_of[m] = np.searchsorted(bounds0[:, r], tp.order_row[m], side="right") - 1
    ks = key[order]
    m = len(ks)
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]]) if m else np.zeros(0, np.int64)
    ends = np.r_[starts[1:], m].astype(np.int64)
    assert np.array_equal(tile_of[starts], tile_of[ends - 1]), "a key spans two tiles"
    live = ~np.isin(kind, RETRACT)
    idx = np.arange(m, dtype=np.int64)
    if rule == "all":
        winner = ends - 1
    elif rule == "drop_delete":
        winner = np.where(live[ends - 1], ends - 1, -1)
    elif rule == "ignore_delete":
        newest_live = np.maximum.accumulate(np.where(live, idx, -1)) if m else idx
        w = newest_live[ends - 1] if m else ends
        winner = np.where(w >= starts, w, -1)
    else:
        raise ValueError(rule)
    out = winner >= 0
    tp.plan_rows = np.bincount(tile_of[starts[out]], minlength=n_tiles[0]).astype(np.int64)
    if value_lens is not None:
        lens = np.concatenate([np.asarray(value_lens[r])[row0[r]:] for r in range(k)])[order]
        tp.plan_bytes = np.bincount(tile_of[starts[out]], weights=lens[winner[out]],
                                    minlength=n_tiles[0]).astype(np.int64)
    return tp


# ---- the edges a shape can claim
def edges(tp: TilePlan, start_rows: Optional[Sequence[int]] = None) -> set:
    """Which of the named structural edges the merge reaches."""
    out = set()
    if tp.n_tiles % 2 == 1 and tp.n_tiles > 1:
        out.add("odd_plan_tiles")
    if tp.n_levels >= 3:
        out.add("three_levels")
    if start_rows is not None and any(start_rows) and tp.n_levels >= 1:
        out.add("start_rows_strided")
    if tp.plan_rows is not None:
        rows = tp.emit_rows()
        nz = np.flatnonzero(rows > 0)
        if len(nz) and np.any(rows[: nz[-1]] == 0):
            out.add("zero_row_emit_tile")
        if len(np.unique(tp.out_base() % 32)) >= 8:
            out.add("out_base_residues")
        if tp.plan_bytes is not None:
            b = tp.emit_bytes()
            nzb = np.flatnonzero(b > 0)
            if len(nzb) and np.any((b[: nzb[-1]] == 0) & (rows[: nzb[-1]] > 0)):
                out.add("zero_byte_tile")
    return out
