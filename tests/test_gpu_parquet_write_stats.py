"""Statistics of the files the device encoder writes, against the independent model (tests/stats_reference.py): the
footer's row-group Statistics as pyarrow reads them, pg_parquet_file_column_stats of every column (keys, sequence
number and kind included), WrittenFile.value_stats and the DataFileMeta fields, for the uncompressed and the zstd
encode, with floats compared bit for bit.  Every min / max reported must also bound the values it describes under
Double.compare (soundness).  The layouts put edge values where k_pw_stats can lose them: at the rows where its
256-thread stride turns over, alone in a chunk, in one row group only, just outside an encoded slice.  Needs an H100."""
import ctypes as C
import struct

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import stats_reference as S
from paimon_b200 import _native as N
from paimon_b200.columnar import Column, KeyValueBatch
from paimon_b200.compact_rewriter import KeyValueDataFileWriter, MergeTreeCompactRewriter, file_column_names
from paimon_b200.merge_function import AggregateMergeFunction
from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition
from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType, is_varlen

from parquet_util import arrow_to_batch, write_kv_parquet
from test_stats_reference_cpu import (EDGES, I64_MAX, ORDINARY, column, draw, is_nan_edge, make_batch, mixed_values,
                                      stats_schema)

pytestmark = pytest.mark.gpu

SMALL = dict(page_rows=64, row_group_rows=256)
WRITERS = [dict(), SMALL]
FLOATS = (PhysicalType.FLOAT, PhysicalType.DOUBLE)


# ---------------------------------------------------------------------------------------------- surfaces

def _device_encode(lib, h, n_cols, names, row0, n, codec, opts):
    """pg_parquet_encode (codec None) or pg_parquet_encode_compressed -> (file bytes, pg_file_meta,
    [(null_count, has_min_max, min8, max8)] of every column)."""
    fh = C.c_uint64(0)
    if codec is None:
        N.check(lib.pg_parquet_encode(h, names, row0, n, C.byref(opts), C.byref(fh)))
    else:
        N.check(lib.pg_parquet_encode_compressed(h, names, row0, n, C.byref(opts), codec, 1, C.byref(fh)))
    try:
        meta = N.PgFileMeta()
        N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
        buf = np.zeros(max(meta.file_bytes, 1), np.uint8)
        N.check(lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
        cols = []
        for c in range(n_cols):
            nulls, has = C.c_int64(0), C.c_int32(0)
            mn, mx = np.zeros(1, np.int64), np.zeros(1, np.int64)
            N.check(lib.pg_parquet_file_column_stats(fh.value, c, C.byref(nulls), C.byref(has), mn.ctypes.data,
                                                     mx.ctypes.data))
            cols.append((int(nulls.value), bool(has.value), mn.tobytes(), mx.tobytes()))
        return bytes(buf[: meta.file_bytes]), meta, cols
    finally:
        lib.pg_parquet_file_free(fh.value)


def footer_of(file_bytes, types):
    """[row group][column] ChunkStats as pyarrow reads them from the footer."""
    md = pq.ParquetFile(pa.BufferReader(file_bytes)).metadata
    out = []
    for g in range(md.num_row_groups):
        row = []
        for c, t in enumerate(types):
            cs = md.row_group(g).column(c).statistics
            assert cs is not None and cs.has_null_count, f"row group {g} column {c}: no statistics"
            if cs.has_min_max:
                row.append(S.ChunkStats(cs.null_count, S.footer_bytes(t, cs.min), S.footer_bytes(t, cs.max)))
            else:
                row.append(S.ChunkStats(cs.null_count, None, None))
        out.append(row)
    return out


def _raw_of_model(t, st: S.FileColStats):
    """A model FileColStats as pg_parquet_file_column_stats reports it: (null_count, has, min8, max8)."""
    if st.min is None:
        return st.null_count, False, None, None
    pack = (lambda v: struct.pack("<d", v)) if t in FLOATS else (lambda v: struct.pack("<q", int(v)))
    return st.null_count, True, pack(st.min), pack(st.max)


def _key(t, v):
    """A SimpleColStats value for an exact comparison: floats by their bits, bool apart from int."""
    if v is None:
        return None
    if t in FLOATS:
        return "f", struct.pack("<d", v)
    return type(v).__name__, v


def _value(t, b8):
    return struct.unpack("<d", b8)[0] if t in FLOATS else struct.unpack("<q", b8)[0]


def check_statistics(schema, batch, tmp_path, row0=0, n=None, **writer_args):
    """Encode rows [row0, row0 + n) of `batch` on the device with both codecs, through the C ABI and through
    KeyValueDataFileWriter, and hold every statistics surface to the model.  Returns the model's footer stats."""
    n = batch.n_rows - row0 if n is None else n
    types = schema.physical_types()
    nk = schema.n_key
    want_footer = S.footer_stats(batch, row0, n, **writer_args)
    want_file = S.file_stats(batch, row0, n)
    want_meta = S.data_file_meta(batch, row0, n)
    lib = N.init(0)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[x.encode() for x in names])
    opts = N.PgParquetWriteOptions(writer_args.get("row_group_rows", 0), writer_args.get("page_rows", 0))
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    try:
        h = rd._open(sh.handle)
        encoded = {codec: _device_encode(lib, h, schema.n_cols, arr, row0, n, codec, opts) for codec in (None, 6)}
        written = {}
        for comp in ("none", "zstd"):
            path = tmp_path / f"{comp}.parquet"
            written[comp] = KeyValueDataFileWriter(schema, str(path), 0, compression=comp, **writer_args).write(h, row0, n)
            assert path.read_bytes() == encoded[None if comp == "none" else 6][0]
    finally:
        rd.close()
        sh.close()

    for codec, (file_bytes, meta, cols) in encoded.items():
        what = "uncompressed" if codec is None else "zstd"
        # footer row-group statistics
        got_footer = footer_of(file_bytes, types)
        assert len(got_footer) == len(want_footer), what
        groups = S.row_groups(n, **writer_args)
        for g, (gg, gw, (a, b)) in enumerate(zip(got_footer, want_footer, groups)):
            for c, (x, w) in enumerate(zip(gg, gw)):
                if x.has_min_max:
                    vals = S.non_null_values(batch.columns[c], row0 + a, row0 + b)
                    bad = S.unsound(types[c], S.value_of(types[c], x.min), S.value_of(types[c], x.max), vals)
                    assert not bad, f"{what}: row group {g} column {names[c]}: {bad[:4]} outside [min, max] = {x}"
                assert x == w, f"{what}: row group {g} column {names[c]}: device {x} model {w}"
        # file-level statistics of every column
        for c, (t, raw, w) in enumerate(zip(types, cols, want_file)):
            nulls, has, mn, mx = raw
            if has and not is_varlen(t):
                vals = S.non_null_values(batch.columns[c], row0, row0 + n)
                bad = S.unsound(t, _value(t, mn), _value(t, mx), vals)
                assert not bad, f"{what}: file column {names[c]}: {bad[:4]} outside [{_value(t, mn)}, {_value(t, mx)}]"
            assert (nulls, has) == _raw_of_model(t, w)[:2], f"{what}: file column {names[c]}: {raw} model {w}"
            if has:
                assert (mn, mx) == _raw_of_model(t, w)[2:], f"{what}: file column {names[c]}: {raw} model {w}"
        # DataFileMeta fields of the C ABI
        assert (meta.n_rows, meta.min_sequence_number, meta.max_sequence_number, meta.delete_row_count) == \
            (want_meta.row_count, want_meta.min_sequence_number, want_meta.max_sequence_number,
             want_meta.delete_row_count), what
    # the writer's SimpleColStats and DataFileMeta
    for comp, w in written.items():
        got = [_key(t, v) for t, s in zip(types[nk + 2:], w.value_stats) for v in (s.min, s.max)]
        exp = [_key(t, v) for t, s in zip(types[nk + 2:], want_file[nk + 2:]) for v in (s.min, s.max)]
        assert got == exp, comp
        assert [s.null_count for s in w.value_stats] == [s.null_count for s in want_file[nk + 2:]], comp
        m = w.meta
        assert S.FileMeta(m.row_count, m.min_sequence_number, m.max_sequence_number, m.delete_row_count, m.min_key,
                          m.max_key) == want_meta, comp
    return want_footer


def _col(schema, logical, nullable=True):
    """Index of the first file column of a logical type in stats_schema()."""
    for c, f in enumerate(schema.file_fields()):
        if f.type == logical and f.nullable == nullable and c >= schema.n_key + 2:
            return c
    raise KeyError(logical)


# ---------------------------------------------------------------------------------------------- layouts

@pytest.mark.parametrize("n", [1, 7, 8, 255, 256, 257, 1000, 4097])
@pytest.mark.parametrize("writer", WRITERS, ids=["default", "small"])
@pytest.mark.parametrize("nan", [False, True], ids=["finite", "nan"])
def test_mixed_edge_values(tmp_path, n, writer, nan):
    """Every row drawn from the edge and ordinary pools of its type, nullable columns about 25 % NULL."""
    schema = stats_schema()
    rng = np.random.default_rng(1000 * n + 10 * bool(writer) + nan)
    check_statistics(schema, make_batch(schema, n, rng, mixed_values(rng, nan=nan)), tmp_path, **writer)


GROUP = 320            # > 257 rows, a multiple of the 64-row pages


@pytest.mark.parametrize("pos", [0, 255, 256, 257, GROUP - 1])
def test_edge_value_alone_at_a_row(tmp_path, pos):
    """Row group g (320 rows) holds edge value g of each column's pool at row `pos`, ordinary values elsewhere:
    the first row, the last thread of the first stride (255), the first rows of the second (256, 257), the last row."""
    schema = stats_schema()
    n_edges = max(len(v) for v in EDGES.values())
    rng = np.random.default_rng(pos)

    def values_of(logical, nullable, n):
        vals = draw(rng, ORDINARY[logical], n)
        valid = rng.random(n) >= 0.1 if nullable else None
        for g in range(n_edges):
            r = g * GROUP + pos
            vals[r] = EDGES[logical][g % len(EDGES[logical])]
            if valid is not None:
                valid[r] = True
        return vals, valid

    want = check_statistics(schema, make_batch(schema, n_edges * GROUP, rng, values_of), tmp_path, page_rows=64,
                            row_group_rows=GROUP)
    d = _col(schema, "DOUBLE")
    assert want[1][d].min == struct.pack("<Q", 0x8000000000000000) and not want[2][d].has_min_max


@pytest.mark.parametrize("n,valid_row", [(8, None), (1000, None), (1, 0), (300, 257), (1000, 999)])
@pytest.mark.parametrize("writer", WRITERS, ids=["default", "small"])
def test_nullable_columns_with_at_most_one_value(tmp_path, n, valid_row, writer):
    """Nullable columns all NULL, or NULL except one row holding a (non-NaN) edge value."""
    schema = stats_schema()
    rng = np.random.default_rng(n + 7 * (valid_row or 0))

    def values_of(logical, nullable, n):
        vals = draw(rng, ORDINARY[logical], n)
        if not nullable:
            return vals, None
        valid = np.zeros(n, bool)
        if valid_row is not None:
            pool = [v for v in EDGES[logical] if not is_nan_edge(logical, v)]
            vals[valid_row] = pool[valid_row % len(pool)]
            valid[valid_row] = True
        return vals, valid

    want = check_statistics(schema, make_batch(schema, n, rng, values_of), tmp_path, **writer)
    end = min(n, 256) if writer else n                 # the first row group
    assert want[0][_col(schema, "BIGINT")].null_count == end - (valid_row is not None and valid_row < end)


@pytest.mark.parametrize("where", ["first", "last"])
def test_nan_in_one_row_group_only(tmp_path, where):
    """1000 rows in row groups of 256: NaNs (quiet, sign bit set, with payload) only in the first or only in the last
    group; the other groups hold zeros, infinities and extremes.  The file has no FLOAT / DOUBLE min / max."""
    schema = stats_schema()
    rng = np.random.default_rng(5 if where == "first" else 6)
    lo, hi = (0, 256) if where == "first" else (768, 1000)

    def values_of(logical, nullable, n):
        finite = [v for v in EDGES[logical] if not is_nan_edge(logical, v)] + ORDINARY[logical]
        vals = draw(rng, finite, n)
        nans = [v for v in EDGES[logical] if is_nan_edge(logical, v)]
        for i, r in enumerate(rng.choice(np.arange(lo, hi), size=min(len(nans) * 2, hi - lo), replace=False)):
            vals[r] = nans[i % len(nans)]
        if nans:
            vals[lo + 1] = nans[0]                     # and one NaN that is surely not NULL
        valid = rng.random(n) >= 0.2 if nullable else None
        if valid is not None:
            valid[lo + 1] = True
        return vals, valid

    batch = make_batch(schema, 1000, rng, values_of)
    want = check_statistics(schema, batch, tmp_path, **SMALL)
    for logical in ("FLOAT", "DOUBLE"):
        for nullable in (True, False):
            c = _col(schema, logical, nullable)
            nan_group = 0 if where == "first" else 3
            assert [g[c].has_min_max for g in want] == [g != nan_group for g in range(4)]
            assert S.file_stats(batch)[c].min is None


ZERO_LAYOUTS = {
    # name: (writer, rows, FLOAT / DOUBLE value of row i, BOOLEAN value of row i)
    "only_pos": (dict(), 300, lambda i: 0.0, lambda i: 1),
    "only_neg": (dict(), 300, lambda i: -0.0, lambda i: 0),
    "pos_one_neg_at_257": (dict(), 300, lambda i: -0.0 if i == 257 else 0.0, lambda i: int(i != 257)),
    "neg_one_pos_at_255": (dict(), 300, lambda i: 0.0 if i == 255 else -0.0, lambda i: int(i == 255)),
    # row groups of 256: +0.0 only / -0.0 only / both / zeros and positives / zeros and negatives
    "groups": (SMALL, 1280, lambda i: [0.0, -0.0, (0.0, -0.0)[i % 2], (0.0, -0.0, 2.5)[i % 3],
                                       (-0.0, 0.0, -2.5)[i % 3]][i // 256],
               lambda i: [1, 0, i % 2, 1, 0][i // 256]),
}


@pytest.mark.parametrize("layout", list(ZERO_LAYOUTS))
def test_signed_zero_chunks(tmp_path, layout):
    """Chunks of only +0.0, only -0.0, and both: the footer min is -0.0 and the max +0.0 whatever zero a warp saw
    first, so that min <= v <= max holds for both zeros; BOOLEAN chunks all true, all false and mixed."""
    writer, n, zero, boolean = ZERO_LAYOUTS[layout]
    schema = stats_schema()
    rng = np.random.default_rng(len(layout))

    def values_of(logical, nullable, n):
        valid = rng.random(n) >= 0.1 if nullable else None
        if logical in ("FLOAT", "DOUBLE"):
            return [zero(i) for i in range(n)], valid
        if logical == "BOOLEAN":
            return [boolean(i) for i in range(n)], valid
        return draw(rng, ORDINARY[logical], n), valid

    want = check_statistics(schema, make_batch(schema, n, rng, values_of), tmp_path, **writer)
    neg0, pos0 = struct.pack("<Q", 0x8000000000000000), bytes(8)
    c = _col(schema, "DOUBLE", False)
    assert want[0][c] == S.ChunkStats(0, neg0, pos0)


@pytest.mark.parametrize("row0,n", [(8, 301), (256, 77), (264, 1001)])
@pytest.mark.parametrize("writer", WRITERS, ids=["default", "small"])
def test_slice_statistics_stay_inside_the_slice(tmp_path, row0, n, writer):
    """KeyValueDataFileWriter.write(h, row0, n): the rows just before row0 and just after row0 + n hold each
    column's extremes, NaNs, NULLs, the sequence number extremes and retract kinds; the inside holds ordinary
    values.  Statistics that read one row too many or too few differ from the model."""
    schema = stats_schema()
    total = row0 + n + 24
    rng = np.random.default_rng(row0 + n)
    before, after = row0 - 1, row0 + n

    def values_of(logical, nullable, total):
        edges = EDGES[logical]
        finite = [v for v in edges if not is_nan_edge(logical, v)]
        vals = draw(rng, edges, total)
        vals[row0:row0 + n] = draw(rng, ORDINARY[logical], n)
        if logical != "STRING":
            vals[before], vals[after] = min(finite), max(finite)
        nans = [v for v in edges if is_nan_edge(logical, v)]
        if nans:
            vals[before - 1], vals[after + 1] = nans[0], nans[-1]
        if not nullable:
            return vals, None
        valid = np.ones(total, bool)
        valid[row0:row0 + n] = rng.random(n) >= 0.1
        valid[[before - 2, after + 2]] = False
        return vals, valid

    batch = make_batch(schema, total, rng, values_of)
    nk = schema.n_key
    seq = rng.integers(1000, 1 << 40, total, dtype=np.int64)
    seq[[before, after]] = [0, I64_MAX]
    kinds = rng.choice(np.array([0, 2], np.int8), total)
    kinds[rng.integers(row0, row0 + n, 5)] = 1
    kinds[[before, after]] = [3, 1]
    batch.columns[nk] = Column(PhysicalType.INT64, seq)
    batch.columns[nk + 1] = Column(PhysicalType.INT8, kinds)
    check_statistics(schema, batch, tmp_path, row0=row0, n=n, **writer)


# ---------------------------------------------------------------------------------------------- end to end

def _e2e_schema():
    vt = RowType((DataField("k", "BIGINT", False), DataField("d", "DOUBLE", True), DataField("f", "FLOAT", True),
                  DataField("i", "INT", True), DataField("t", "TINYINT", True), DataField("b", "BOOLEAN", True),
                  DataField("ts", "TIMESTAMP(6)", True), DataField("dec", "DECIMAL(18,4)", True),
                  DataField("s", "STRING", True)))
    return vt, KeyValueSchema.of(vt, ["k"])


@pytest.mark.parametrize("drop_delete", [False, True])
def test_compaction_output_statistics(tmp_path, drop_delete):
    """Input files carrying the edge values -> MergeTreeCompactRewriter (aggregation: sum over DOUBLE, where
    +inf + -inf makes the merge itself produce NaN; last non-null value elsewhere) with files of at most 400 rows.
    The value_stats, DataFileMeta and footer of every output file equal the model over that file's rows as pyarrow
    reads them back."""
    vt, schema = _e2e_schema()
    logical = [f.type for f in vt.fields]
    rng = np.random.default_rng(31 + drop_delete)
    inf_keys = set(range(1500, 1520))                  # +inf in run 0, -inf in run 1: the sum is NaN
    nan_keys = set(range(2500, 2540))                  # the only keys whose FLOAT inputs may be NaN
    metas, n_runs = [], 4
    for r in range(n_runs):
        keys = np.sort(rng.choice(np.arange(3000), 1500, replace=False))
        if r < 2:
            keys = np.union1d(keys, sorted(inf_keys))
        rows = []
        for i, k in enumerate(keys):
            row = [int(k)]
            for name, lg in zip(vt.field_names()[1:], logical[1:]):
                pool = [v for v in EDGES[lg] + ORDINARY[lg]
                        if not (is_nan_edge(lg, v) and (name == "d" or k not in nan_keys))
                        and not (name == "d" and np.isinf(v))]
                v = pool[rng.integers(0, len(pool))]
                if name == "d" and k in inf_keys and r < 2:
                    v = np.inf if r == 0 else -np.inf
                nullable = vt.fields[vt.field_names().index(name)].nullable
                row.append(None if nullable and rng.random() < 0.15 and not (name == "d" and k in inf_keys) else v)
            kind = 0 if k in inf_keys and r < 2 else int(rng.choice([0, 0, 0, 2, 1, 3]))
            rows.append((int(k), r * 100_000 + i, kind, *row))
        types = schema.physical_types()
        cols = [column(t, [row[c] if row[c] is not None else (0 if not is_varlen(t) else "") for row in rows],
                       np.array([row[c] is not None for row in rows])) for c, t in enumerate(types)]
        batch = KeyValueBatch(schema, cols)
        path = str(tmp_path / f"in-{r}.parquet")
        write_kv_parquet(batch, path, use_dictionary=(r % 2 == 0))
        metas.append(DataFileMeta(path, 0, batch.n_rows, int(keys[0]), int(keys[-1]), level=0))
    factory = AggregateMergeFunction.factory({"fields.d.aggregate-function": "sum"}, vt, ["k"])
    out = tmp_path / "out"
    out.mkdir()
    rewriter = MergeTreeCompactRewriter(schema, factory, str(out), target_file_rows=400, page_rows=64,
                                        row_group_rows=128)
    result = rewriter.rewrite_compaction(3, drop_delete, IntervalPartition(metas).partition())
    assert len(result.written) >= 5
    nk = schema.n_key
    types = schema.physical_types()
    d = nk + 2 + 1
    saw_nan_file = saw_finite_file = False
    for w in result.written:
        back = arrow_to_batch(schema, pq.read_table(w.meta.file_name))
        want = S.file_stats(back)
        got = [_key(t, v) for t, s in zip(types[nk + 2:], w.value_stats) for v in (s.min, s.max)]
        exp = [_key(t, v) for t, s in zip(types[nk + 2:], want[nk + 2:]) for v in (s.min, s.max)]
        assert got == exp, w.meta.file_name
        assert [s.null_count for s in w.value_stats] == [s.null_count for s in want[nk + 2:]]
        m = w.meta
        assert S.FileMeta(m.row_count, m.min_sequence_number, m.max_sequence_number, m.delete_row_count, m.min_key,
                          m.max_key) == S.data_file_meta(back), w.meta.file_name
        with open(w.meta.file_name, "rb") as f:
            assert footer_of(f.read(), types) == S.footer_stats(back, page_rows=64, row_group_rows=128)
        dvals = S.non_null_values(back.columns[d], 0, back.n_rows)
        if np.isnan(dvals).any():
            saw_nan_file = True
            assert want[d].min is None
        elif len(dvals):
            saw_finite_file = True
            assert not S.unsound(PhysicalType.DOUBLE, w.value_stats[1].min, w.value_stats[1].max, dvals)
    assert saw_nan_file and saw_finite_file
