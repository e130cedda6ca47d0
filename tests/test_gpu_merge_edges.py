"""The device merge at the edges of its tile structure, compared bit for bit with the oracle's LoserTree merge.

Every case also checks that the merge's level and tile counts equal those of the tile model (merge_tiles.py), so
each case provably reaches the structure it is named for: full overlap at the tile bound, disjoint and skewed runs,
key types at their extremes, non-exact keys over three levels, plan and emit tiles without output, var-len tiles
without bytes, start rows and slices, and the 2 GiB limit of a var-len output column.  Needs an H100."""
import gc

import numpy as np
import pytest

from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200.columnar import Column, KeyValueBatch
from paimon_b200.merge_function import (AggregateMergeFunction, DeduplicateMergeFunction, FirstRowMergeFunction,
                                        PartialUpdateMergeFunction)
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader, fetch_slice, merge_runs, slice_rows
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType, numpy_dtype

import merge_shapes as ms
import merge_tiles as mt

pytestmark = pytest.mark.gpu
P = PhysicalType


def oracle_runs(shape):
    if not shape.start_rows:
        return shape.runs
    return [slice_rows(r, s, r.n_rows) for r, s in zip(shape.runs, shape.start_rows)]


def merge_and_check(shape, spec, tp=None, slices=None):
    """Merge on the device, compare with the oracle and the model; returns the merged batch.  `slices(n_rows)`
    gives row ranges of the merged batch that are also fetched through slice views."""
    tp = tp or shape.plan()
    readers = [SortedRunReader(shape.schema, b) for b in shape.runs]
    rd = SortMergeReader(readers, spec, start_rows=shape.start_rows)
    try:
        rd.execute()
        st = rd.stats()
        got = rd.fetch()
        sliced = [(lo, hi, fetch_slice(shape.schema, rd._merge_h, lo, hi)) for lo, hi in (slices or (lambda n: ()))(got.n_rows)]
    finally:
        rd.close()
    want = pyoracle.merge(shape.schema, spec, oracle_runs(shape), pyoracle.SORT_LOSER_TREE)
    assert got.equals(want), got.first_difference(want)
    assert (st.n_levels, st.n_tiles) == (tp.n_levels, tp.n_tiles)
    if tp.plan_rows is not None and shape.rule != "all":
        assert got.n_rows == int(tp.plan_rows.sum())
    for lo, hi, part in sliced:
        w = slice_rows(want, lo, hi)
        assert part.equals(w), (lo, hi, part.first_difference(w))
    return got


def specs_for(shape):
    vt = shape.schema.value_type
    return {
        "dedup": DeduplicateMergeFunction.factory().create(),
        "pu": PartialUpdateMergeFunction.factory({}, vt, ["k"]).create(),
        "agg_double_sum": AggregateMergeFunction.factory({"fields.d.aggregate-function": "sum",
                                                          "fields.s.aggregate-function": "max"}, vt, ["k"]).create(),
    }


# ---- 1. full overlap
@pytest.mark.parametrize("spec_name", ["dedup", "pu", "agg_double_sum"])
@pytest.mark.parametrize("k,n", ms.FULL_OVERLAP)
def test_full_overlap(k, n, spec_name):
    """Every key in every run, k = 1..32 and 0 to 3 levels; k = 32 at 640 K rows is the tight tile bound, and the
    DOUBLE sum folds 32 members in sequence order."""
    sh = ms.full_overlap(k, n)
    tp = sh.plan()
    assert tp.largest_tile <= mt.tile_bound(k)
    merge_and_check(sh, specs_for(sh)[spec_name], tp)


# ---- 2. + 3. disjoint, interleaved, banded, skewed runs
@pytest.mark.parametrize("builder", [ms.disjoint, ms.interleaved, ms.banded, ms.skew, ms.stride_lengths],
                         ids=lambda b: b.__name__)
def test_run_layouts(builder):
    sh = builder()
    merge_and_check(sh, DeduplicateMergeFunction.factory().create())
    merge_and_check(sh, specs_for(sh)["agg_double_sum"])


# ---- 4. key types at their extremes
INT_TYPES = {"TINYINT": (np.int8, P.INT8), "SMALLINT": (np.int16, P.INT16), "INT": (np.int32, P.INT32),
             "BIGINT": (np.int64, P.INT64), "BOOLEAN": (np.uint8, P.BOOL), "DATE": (np.int32, P.INT32),
             "TIMESTAMP(3)": (np.int64, P.INT64), "DECIMAL(18, 2)": (np.int64, P.INT64)}


def pool_shape(name, key_fields, pool, k=3, frac=0.6, seed=0, always=()):
    """Runs that each take a random sorted subset of `pool` (key tuples sorted in the true key order); the pool
    entries listed in `always` are in every run."""
    rng = np.random.default_rng(seed)
    schema = ms.value_schema(tuple(key_fields), [f.name for f in key_fields])
    n = len(pool)
    picks = []
    for r in range(k):
        m = rng.random(n) < frac
        m[list(always)] = True
        picks.append(np.flatnonzero(m))
    seqs = ms.unique_seqs([len(p) for p in picks], seed)
    runs = []
    for r, idx in enumerate(picks):
        cols = []
        for f_i, f in enumerate(key_fields):
            vals = [pool[i][f_i] for i in idx]
            pt = PhysicalType(int(f.physical))
            if pt in (P.STRING, P.BINARY):
                cols.append(Column.from_pylist(pt, vals))
            else:
                cols.append(Column(pt, np.array(vals, dtype=numpy_dtype(pt))))
        runs.append(ms.run_batch(schema, cols, seqs[r], np.zeros(len(idx), np.int8), rng))
    return ms.Shape(name, schema, runs, [p.astype(np.int64) for p in picks])


def sorted_pool(tuples):
    return sorted(set(tuples), key=mt.true_key)


@pytest.mark.parametrize("logical", sorted(INT_TYPES))
def test_single_integer_key_extremes(logical):
    """MIN, MAX, -1, 0 and 1 of every integer key type (the sign flip of the key's order-preserving image), in
    every run; DATE, TIMESTAMP(3) and DECIMAL(18, 2) share the integer path."""
    dt, _ = INT_TYPES[logical]
    rng = np.random.default_rng(len(logical))
    if logical == "BOOLEAN":
        extremes, rest = [0, 1], []
    else:
        info = np.iinfo(dt)
        extremes = [int(info.min), int(info.max), -1, 0, 1]
        rest = rng.integers(int(info.min), int(info.max), 30000, dtype=np.int64, endpoint=True).tolist()
    pool = sorted_pool([(x,) for x in extremes + rest])
    always = [i for i, t in enumerate(pool) if t[0] in extremes]
    sh = pool_shape(logical, [DataField("k", logical, False)], pool, seed=3, always=always)
    got = merge_and_check(sh, DeduplicateMergeFunction.factory().create())
    keys = got.columns[0].data[: got.n_rows].astype(np.int64)
    assert set(extremes) <= set(keys.tolist())


def composite_pool(kind, n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        if kind == "exact8":
            out.append((int(rng.integers(0, 2)), int(rng.integers(-128, 128)), int(rng.integers(-4, 4)),
                        int(rng.integers(-2 ** 31, 2 ** 31))))
        elif kind == "nine_bytes":
            out.append((int(rng.integers(-128, 128)), int(rng.choice([-2 ** 63, -1, 0, 1, 2 ** 63 - 1]))
                        if rng.random() < 0.1 else int(rng.integers(-2 ** 63, 2 ** 63 - 1))))
        else:
            s = rng.choice(["", "a", "ab", "abcdefgh", "abcdefghi", "b\x00", "\x7f"])
            out.append((int(rng.integers(-2000, 2000)), str(s), int(rng.integers(-2, 2)), int(rng.integers(-50, 50))))
    return sorted_pool(out)


COMPOSITES = {
    "exact8": [DataField("a", "BOOLEAN", False), DataField("b", "TINYINT", False), DataField("c", "SMALLINT", False),
               DataField("e", "INT", False)],
    "nine_bytes": [DataField("a", "TINYINT", False), DataField("b", "BIGINT", False)],
    "varlen_not_last": [DataField("a", "INT", False), DataField("b", "STRING", False),
                        DataField("c", "SMALLINT", False), DataField("e", "BIGINT", False)],
}


@pytest.mark.parametrize("kind", sorted(COMPOSITES))
def test_composite_keys(kind):
    """(BOOLEAN, TINYINT, SMALLINT, INT) is exactly 8 bytes (exact) with negatives in every field; (TINYINT, BIGINT)
    is 9 bytes (non-exact); (INT, STRING, SMALLINT, BIGINT) has a var-len field that is not last."""
    pool = composite_pool(kind, 60000, 5)
    sh = pool_shape(kind, COMPOSITES[kind], pool, seed=6)
    assert sh.plan().n_levels >= 2
    merge_and_check(sh, DeduplicateMergeFunction.factory().create())


def test_five_field_key_is_refused():
    fields = tuple(DataField(f"k{i}", "INT", False) for i in range(5)) + (DataField("v", "BIGINT", True),)
    schema = KeyValueSchema.of(RowType(fields), [f"k{i}" for i in range(5)])
    run = KeyValueBatch.from_rows(schema, [(1, 2, 3, 4, 5, 1, 0, 1, 2, 3, 4, 5, 7)])
    with pytest.raises(N.UnsupportedOnDevice, match="more than 4 primary-key fields"):
        merge_runs(schema, DeduplicateMergeFunction.factory().create(), [run, run])


# ---- 5. non-exact keys over three levels
@pytest.mark.parametrize("builder", [ms.changing_prefixes, ms.binary_high_bytes], ids=lambda b: b.__name__)
def test_non_exact_keys_three_levels(builder):
    sh = builder()
    tp = sh.plan()
    assert tp.n_levels >= 3
    merge_and_check(sh, DeduplicateMergeFunction.factory().create(), tp)


# ---- 6. empty output
def test_delete_ranges_drop_delete():
    sh = ms.delete_ranges()
    merge_and_check(sh, DeduplicateMergeFunction.factory().create().with_drop_delete())


def test_delete_ranges_partial_update_remove_on_delete():
    sh = ms.delete_ranges(rod=True)
    spec = PartialUpdateMergeFunction.factory({"partial-update.remove-record-on-delete": "true"},
                                              sh.schema.value_type, ["k"]).create().with_drop_delete()
    merge_and_check(sh, spec)


@pytest.mark.parametrize("engine", ["dedup", "first_row"])
def test_retract_only_groups_ignore_delete(engine):
    sh = ms.retract_only_groups()
    f = DeduplicateMergeFunction if engine == "dedup" else FirstRowMergeFunction
    merge_and_check(sh, f.factory({"ignore-delete": "true"}).create())


def test_whole_output_empty():
    sh = ms.all_deleted()
    got = merge_and_check(sh, DeduplicateMergeFunction.factory().create().with_drop_delete())
    assert got.n_rows == 0
    s = got.value_column(3)
    assert list(np.asarray(s.offsets[:1])) == [0] and len(s.data) == 0


# ---- 7. var-len look-back
def test_null_and_empty_string_ranges():
    sh = ms.null_and_empty_ranges()
    tp = sh.plan()
    assert "zero_byte_tile" in mt.edges(tp)
    merge_and_check(sh, DeduplicateMergeFunction.factory().create(), tp)
    merge_and_check(sh, specs_for(sh)["pu"], tp)


def test_one_16MiB_value():
    sh = ms.one_huge_value()
    got = merge_and_check(sh, DeduplicateMergeFunction.factory().create())
    s = got.value_column(3)
    assert int(np.diff(np.asarray(s.offsets, np.int64)).max()) == 16 << 20


def test_single_run_two_string_columns():
    """k = 1 at 200 K rows: the var-len scratch in the upper half of a stage is tightest."""
    vt = RowType((DataField("k", "BIGINT", False), DataField("s1", "STRING", True), DataField("s2", "STRING", True)))
    schema = KeyValueSchema.of(vt, ["k"])
    n = 200_000
    rng = np.random.default_rng(15)
    keys = Column(P.INT64, np.arange(n, dtype=np.int64) * 3)
    lens = np.where((np.arange(n) // 3000) % 5 == 2, 0, rng.integers(0, 41, n))
    s1 = ms.str_column(lens, 1, rng.random(n) >= 0.1)
    s2 = ms.str_column(rng.integers(0, 9, n), 2, rng.random(n) >= 0.5)
    run = KeyValueBatch(schema, [keys, Column(P.INT64, np.arange(n, dtype=np.int64)), Column(P.INT8, np.zeros(n, np.int8)),
                                 keys, s1, s2])
    sh = ms.Shape("k1_two_strings", schema, [run], [keys.data])
    merge_and_check(sh, DeduplicateMergeFunction.factory().create())


# ---- 8. start rows and slices
def test_start_rows_and_slices():
    sh = ms.start_rows_shape()
    tp = sh.plan()
    assert tp.n_levels >= 2
    def slices(n):
        return [(0, 1), (1, 33), (7, 4103), (n // 2 + 5, n // 2 + 70005), (n - 31, n)]
    merge_and_check(sh, DeduplicateMergeFunction.factory().create(), tp, slices)
    merge_and_check(sh, specs_for(sh)["agg_double_sum"], tp)


# ---- 9. the 2 GiB limit of a var-len output column
BIN_SCHEMA = KeyValueSchema.of(RowType((DataField("k", "BIGINT", False), DataField("b", "BINARY", True))), ["k"])


def fill_byte(j):
    return (j * 37 + 11) & 0xFF


def big_run(keys, lens, seq0, tag=0):
    """A run whose value j is `lens[j]` bytes of one byte value, with its 8-byte index written at its front."""
    keys = np.asarray(keys, np.int64)
    lens = np.asarray(lens, np.int64)
    offs = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    assert offs[-1] < 2 ** 31
    data = np.empty(int(offs[-1]), np.uint8)
    for j in range(len(lens)):
        a, b = int(offs[j]), int(offs[j + 1])
        data[a:b] = fill_byte(int(keys[j]) + tag)
        if b - a >= 8:
            data[a:a + 8] = np.frombuffer(np.int64(keys[j]).tobytes(), np.uint8)
    n = len(keys)
    kc = Column(P.INT64, keys)
    return KeyValueBatch(BIN_SCHEMA, [kc, Column(P.INT64, np.arange(n, dtype=np.int64) + seq0),
                                      Column(P.INT8, np.zeros(n, np.int8)), kc,
                                      Column(P.BINARY, data, offs.astype(np.int32))])


def check_big_output(got, keys, lens, tag=0):
    keys = np.asarray(keys, np.int64)
    lens = np.asarray(lens, np.int64)
    assert got.n_rows == len(keys)
    assert np.array_equal(got.columns[0].data[: len(keys)], keys)
    c = got.value_column(1)
    want_offs = np.zeros(len(keys) + 1, np.int64)
    np.cumsum(lens, out=want_offs[1:])
    assert np.array_equal(np.asarray(c.offsets[: len(keys) + 1], np.int64), want_offs)
    for j in range(len(keys)):
        a, b = int(want_offs[j]), int(want_offs[j + 1])
        body = a
        if b - a >= 8:
            assert np.frombuffer(c.data[a:a + 8].tobytes(), np.int64)[0] == keys[j]
            body = a + 8
        assert np.all(c.data[body:b] == fill_byte(int(keys[j]) + tag))


def run_merge(runs, spec=None):
    spec = spec or DeduplicateMergeFunction.factory().create()
    rd = SortMergeReader([SortedRunReader(BIN_SCHEMA, b) for b in runs], spec)
    return rd


def test_payload_of_exactly_2GiB_minus_1_is_accepted():
    """Two runs with disjoint keys, one tile: the in-tile byte positions reach 2^31 - 1."""
    v = 1 << 26
    keys = np.arange(32)
    lens = [v] * 31 + [v - 1]
    runs = [big_run(keys[:16], lens[:16], 0), big_run(keys[16:], lens[16:], 100)]
    rd = run_merge(runs)
    del runs
    gc.collect()
    try:
        rd.execute()
        got = rd.fetch()
    finally:
        rd.close()
    assert int(got.value_column(1).offsets[32]) == 2 ** 31 - 1
    check_big_output(got, keys, lens)


def test_payload_of_2GiB_over_several_tiles_is_refused():
    v = 1 << 17
    runs = [big_run(np.arange(8192) * 2, [v] * 8192, 0), big_run(np.arange(8192) * 2 + 1, [v] * 8192, 10 ** 6)]
    rd = run_merge(runs)
    del runs
    gc.collect()
    try:
        with pytest.raises(N.PaimonGpuError, match="a var-len column exceeds 2 GiB of payload") as e:
            rd.execute()
        assert e.value.status == 5                              # PG_ERR_INTERNAL
    finally:
        rd.close()


def test_inputs_above_2GiB_with_a_smaller_output_are_accepted():
    """The refusal is on the output: deduplicate keeps the newer short values of inputs summing past 2 GiB."""
    n, v = 8192, 1 << 17
    keys = np.arange(n)
    short = (keys % 23) + 1
    runs = [big_run(keys, [v] * n, 0), big_run(keys, [v] * n, n), big_run(keys, short, 2 * n, tag=1)]
    assert sum(int(r.value_column(1).offsets[-1]) for r in runs) > 2 ** 31
    rd = run_merge(runs)
    del runs
    gc.collect()
    try:
        rd.execute()
        got = rd.fetch()
    finally:
        rd.close()
    check_big_output(got, keys, short, tag=1)


def test_one_emit_tile_above_2GiB_is_refused_and_the_handle_recovers():
    """2200 values of 1 MiB with disjoint keys are two plan tiles, so one emit tile holds 2.2 GiB: refused without a
    store past the output buffer; the same handle then merges a small input correctly."""
    v = 1 << 20
    runs = [big_run(np.arange(1100) * 2, [v] * 1100, 0), big_run(np.arange(1100) * 2 + 1, [v] * 1100, 5000)]
    assert mt.plan([r.columns[0].data for r in runs]).n_tiles == 2
    rd = run_merge(runs)
    del runs
    gc.collect()
    try:
        with pytest.raises(N.PaimonGpuError, match="a var-len column exceeds 2 GiB of payload") as e:
            rd.execute()
        assert e.value.status == 5
        small = [big_run(np.arange(0, 6000, 3), np.arange(2000) % 41, 0),
                 big_run(np.arange(0, 6000, 2), np.arange(3000) % 13, 10 ** 5, tag=2)]
        big_readers = rd.readers
        rd.rebind([SortedRunReader(BIN_SCHEMA, b) for b in small])
        for r in big_readers:                                  # the merge no longer holds them: free them now
            r.close()
        rd.execute()
        got = rd.fetch()
    finally:
        rd.close()
    want = pyoracle.merge(BIN_SCHEMA, DeduplicateMergeFunction.factory().create(), small, pyoracle.SORT_LOSER_TREE)
    assert got.equals(want), got.first_difference(want)


# ---- one handle rebound to a larger input that needs every optional workspace region, then to a smaller one

GROUP_VT = RowType((DataField("k", "STRING", False), DataField("g", "BIGINT", True), DataField("v", "BIGINT", True),
                    DataField("s", "STRING", True)))
GROUP_SCHEMA = KeyValueSchema.of(GROUP_VT, ["k"])


def group_runs(n_keys, n_runs, seed):
    """String keys sharing a prefix (non-exact: the key-prefix skip), a sequence group whose field sums (group plan and
    group aggregates) and a var-len column (look-back state)."""
    rng = np.random.default_rng(seed)
    rows_of_run = [[] for _ in range(n_runs)]
    seq = 0
    for key in range(n_keys):
        k = f"user_{key:07d}"
        for r in sorted(rng.choice(n_runs, size=int(rng.integers(1, n_runs + 1)), replace=False)):
            seq += 1
            g = None if rng.random() < 0.2 else int(rng.integers(0, 5))
            v = None if rng.random() < 0.2 else int(rng.integers(-1000, 1000))
            s = None if rng.random() < 0.2 else "x" * int(rng.integers(0, 24))
            rows_of_run[r].append((k, seq, 0, k, g, v, s))
    return [KeyValueBatch.from_rows(GROUP_SCHEMA, rows) for rows in rows_of_run if rows]


def test_rebind_to_a_larger_input_with_every_workspace_region_and_back():
    spec = PartialUpdateMergeFunction.factory({"fields.g.sequence-group": "v", "fields.v.aggregate-function": "sum"},
                                              GROUP_VT, ["k"]).create()
    inputs = [group_runs(500, 3, seed=1), group_runs(40_000, 4, seed=2), group_runs(300, 2, seed=3)]
    rd = SortMergeReader([SortedRunReader(GROUP_SCHEMA, b) for b in inputs[0]], spec)
    try:
        for i, runs in enumerate(inputs):
            if i:
                previous = rd.readers
                rd.rebind([SortedRunReader(GROUP_SCHEMA, b) for b in runs])
                for r in previous:                             # the merge no longer holds them: free them now
                    r.close()
            rd.execute()
            got = rd.fetch()
            if i == 1:
                assert rd.stats().n_levels >= 2
            want = pyoracle.merge(GROUP_SCHEMA, spec, runs, pyoracle.SORT_LOSER_TREE)
            assert got.equals(want), (i, got.first_difference(want))
    finally:
        rd.close()
