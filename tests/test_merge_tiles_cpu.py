"""The tile model of merge_tiles.py against the oracle's merge order, the tile bound it must respect, and the
structural edges every GPU edge-case shape (merge_shapes.py) claims to reach.  Runs without a GPU."""
import numpy as np
import pytest

from oracle import pyoracle
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.sort_merge_reader import slice_rows

import merge_shapes as ms
import merge_tiles as mt

SMALL = [(ms.full_overlap, dict(k=k, n=n)) for k, n in [(1, 300), (2, 2100), (3, 900), (17, 500), (31, 80), (32, 140)]] + [
    (ms.disjoint, dict(m=700)), (ms.interleaved, dict(m=700)), (ms.banded, dict(m=700)), (ms.skew, dict(big=9000)),
    (ms.stride_lengths, {}), (ms.delete_ranges, dict(n=3000, block=400)), (ms.retract_only_groups, dict(n=2000)),
    (ms.all_deleted, dict(n=700)), (ms.null_and_empty_ranges, dict(n=3000, block=300)),
    (ms.start_rows_shape, dict(m=1500)), (ms.changing_prefixes, dict(m=1500)), (ms.binary_high_bytes, dict(m=1200)),
]


def _id(case):
    b, kw = case
    return b.__name__ + "".join(f"_{k}{v}" for k, v in kw.items())


def oracle_runs(shape):
    """The runs as the oracle sees them: rows before a start row removed."""
    if not shape.start_rows:
        return shape.runs
    return [slice_rows(r, s, r.n_rows) for r, s in zip(shape.runs, shape.start_rows)]


@pytest.mark.parametrize("case", SMALL, ids=_id)
def test_model_order_equals_loser_tree(case):
    builder, kw = case
    sh = builder(**kw)
    tp = sh.plan()
    runs = oracle_runs(sh)
    spec = DeduplicateMergeFunction.factory().create()
    want_run, want_row = pyoracle.merge_order(sh.schema, spec, runs, pyoracle.SORT_LOSER_TREE)
    off = np.array(sh.start_rows or [0] * len(runs), np.int64)
    assert np.array_equal(tp.order_run, want_run)
    assert np.array_equal(tp.order_row, want_row + off[want_run])
    assert tp.largest_tile <= mt.tile_bound(tp.k)
    # every merged row lies in the plan tile the model gives it, and tiles partition the rows
    sizes = np.diff(tp.bounds0, axis=0).sum(axis=1)
    assert sizes.sum() == sum(r.n_rows for r in runs)


@pytest.mark.parametrize("case", [c for c in SMALL if c[0] in (ms.delete_ranges, ms.retract_only_groups,
                                                              ms.all_deleted, ms.null_and_empty_ranges)], ids=_id)
def test_model_output_counts_equal_oracle(case):
    """Per plan tile rows (and bytes) of the model's output rule, against the oracle's merged result."""
    builder, kw = case
    sh = builder(**kw)
    tp = sh.plan()
    opts = {"ignore-delete": "true"} if sh.rule == "ignore_delete" else {}
    spec = DeduplicateMergeFunction.factory(opts).create()
    if sh.rule == "drop_delete":
        spec = spec.with_drop_delete()
    want = pyoracle.merge(sh.schema, spec, sh.runs, pyoracle.SORT_LOSER_TREE)
    assert tp.plan_rows.sum() == want.n_rows
    if tp.plan_bytes is not None:
        s = want.value_column(sh.lens_col)
        assert tp.plan_bytes.sum() == int(s.offsets[want.n_rows]) - int(s.offsets[0])
    # the key of every output row sits in the tile the model counted it in
    keys = want.columns[0].data[: want.n_rows]
    per_tile = []
    for t in range(tp.n_tiles):
        lo = np.concatenate([sh.ordinals[r][tp.bounds0[t, r]:tp.bounds0[t + 1, r]] for r in range(len(sh.runs))])
        per_tile.append(np.isin(keys, lo).sum())
    assert np.array_equal(np.array(per_tile), tp.plan_rows)


def _sweep_shapes(seed):
    rng = np.random.default_rng(seed)
    for k in range(1, 33):
        for kind in ("full", "disjoint", "random"):
            base = [16 ** l + d for l in (1, 2, 3) for d in (-1, 0, 1)]
            lens = [int(rng.choice(base)) for _ in range(k)]
            if kind == "full":
                n = int(rng.choice(base))
                ords = [np.arange(n, dtype=np.int64)] * k
            elif kind == "disjoint":
                ords, at = [], 0
                for n in lens:
                    ords.append(np.arange(at, at + n, dtype=np.int64))
                    at += n
            else:
                ords = [np.sort(rng.choice(5000, min(n, 4000), replace=False)).astype(np.int64) for n in lens]
            starts = [int(rng.integers(0, max(len(o) // 2, 1))) if rng.random() < 0.5 else 0 for o in ords]
            yield k, kind, ords, None
            yield k, kind, ords, starts


def test_tile_bound_sweep():
    """Largest tile <= 2032 - k over k = 1..32: full overlap, disjoint and random runs whose lengths sit at
    16^l - 1, 16^l and 16^l + 1, with and without start rows."""
    worst = {}
    for k, kind, ords, starts in _sweep_shapes(21):
        tp = mt.plan(ords, starts)
        assert tp.largest_tile <= mt.tile_bound(tp.k), (k, kind, starts, tp.largest_tile)
        worst[k] = max(worst.get(k, 0), tp.largest_tile)
    assert mt.tile_bound(32) == 2000 and mt.tile_bound(1) == 2031
    assert len(worst) == 32


def test_full_overlap_bound_at_three_levels():
    sh = ms.full_overlap(32, 20000)
    tp = mt.plan(sh.ordinals)
    assert tp.n_levels == 3 and tp.largest_tile <= mt.tile_bound(32)


@pytest.mark.parametrize("case", ms.gpu_shapes(), ids=_id)
def test_gpu_shape_reaches_claimed_edges(case):
    """What each GPU edge case is named for is confirmed by the model, so that a change of a generator cannot
    silently stop reaching it."""
    builder, kw = case
    sh = builder(**kw)
    tp = sh.plan()
    got = mt.edges(tp, sh.start_rows)
    assert sh.claims <= got, (sh.name, sh.claims - got)
    assert tp.largest_tile <= mt.tile_bound(tp.k)
