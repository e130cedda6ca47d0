"""The statistics model (tests/stats_reference.py) on the CPU: hand-worked answers for every rule, and agreement with
pyarrow's Parquet writer on NaN-free data with zeros, infinities and integer extremes.  The value pools and batch
builders here are shared with test_gpu_parquet_write_stats.py, which holds the device encoder to the same model."""
import struct

import numpy as np
import pyarrow.parquet as pq
import pytest

import stats_reference as S
from paimon_b200.columnar import Column, KeyValueBatch, pack_validity
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType, is_varlen, numpy_dtype

from parquet_util import to_arrow

F32 = lambda bits: np.frombuffer(struct.pack("<I", bits), np.float32)[0]      # noqa: E731
F64 = lambda bits: np.frombuffer(struct.pack("<Q", bits), np.float64)[0]      # noqa: E731
NEG0_F64 = struct.pack("<Q", 0x8000000000000000)
POS0_F64 = bytes(8)

# ---------------------------------------------------------------------------------------------- value pools
# EDGES[type]: the values where statistics go wrong; ORDINARY[type]: a narrow band strictly inside them, so that an
# edge value among ordinary ones is the chunk's min or max (or, for NaN, removes both).

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
EDGES = {
    "TINYINT": [-128, 127, 0, -1],
    "SMALLINT": [-32768, 32767, 0, -1],
    "INT": [-(1 << 31), (1 << 31) - 1, 0, -1],
    "BIGINT": [I64_MIN, I64_MAX, 0, -1],
    "FLOAT": [F32(0x00000000), F32(0x80000000), F32(0x7fc00000), F32(0xffc00000), F32(0x7fa00001),
              np.float32(np.inf), np.float32(-np.inf), F32(0x00000001), F32(0x80000001), F32(0x7f7fffff),
              F32(0xff7fffff)],
    "DOUBLE": [F64(0), F64(0x8000000000000000), F64(0x7ff8000000000000), F64(0xfff8000000000000),
               F64(0x7ff4000000000123), np.inf, -np.inf, F64(1), F64(0x8000000000000001), F64(0x7fefffffffffffff),
               F64(0xffefffffffffffff)],
    "BOOLEAN": [0, 1],
    "DATE": [-(1 << 31), (1 << 31) - 1, -719162, 2932896, 0],          # 0001-01-01, 9999-12-31, 1970-01-01
    "TIMESTAMP(3)": [I64_MIN, I64_MAX, -62135596800000, 253402300799999, 0],
    "TIMESTAMP(6)": [I64_MIN, I64_MAX, -62135596800000000, 253402300799999999, 0],
    "DECIMAL(5,2)": [-99999, 99999, 0, -1],
    "DECIMAL(18,4)": [-(10 ** 18 - 1), 10 ** 18 - 1, 0, -1],
    "STRING": ["", "\x00", "\U0001f600", "zzzz"],
}
ORDINARY = {
    "TINYINT": [3, 5, 7, 11], "SMALLINT": [300, 301, 517], "INT": [70000, 70001, 123456],
    "BIGINT": [1 << 40, (1 << 40) + 7, 1 << 41], "FLOAT": [1.0, 1.25, 1.5, 1.75], "DOUBLE": [1.0, 1.125, 1.5, 1.875],
    "BOOLEAN": [1], "DATE": [19000, 19001, 19500], "TIMESTAMP(3)": [1700000000000, 1700000000123],
    "TIMESTAMP(6)": [1700000000000000, 1700000000000456], "DECIMAL(5,2)": [1234, 1250, 4321],
    "DECIMAL(18,4)": [12345678901234, 12345678901235], "STRING": ["m", "mm", "paimon"],
}
TYPES = list(EDGES)


def is_nan_edge(logical, v) -> bool:
    return logical in ("FLOAT", "DOUBLE") and v != v


def stats_schema() -> KeyValueSchema:
    """pk BIGINT, then every type of the pools twice: nullable, and NOT NULL (suffix _nn)."""
    fields = [DataField("pk", "BIGINT", False)]
    for i, t in enumerate(TYPES):
        fields += [DataField(f"c{i}", t, True), DataField(f"c{i}_nn", t, False)]
    return KeyValueSchema.of(RowType(tuple(fields)), ["pk"])


def column(t: PhysicalType, values, valid=None) -> Column:
    """A column with the exact bits of `values` (NaN payloads kept); valid = bool mask or None."""
    if is_varlen(t):
        return Column.from_pylist(t, [v if valid is None or valid[i] else None for i, v in enumerate(values)])
    dt = numpy_dtype(t)
    data = np.empty(len(values), dt)
    for i, v in enumerate(values):
        data[i] = v
    vbits = None if valid is None or np.all(valid) else pack_validity(valid)
    return Column(t, data, None, vbits)


def make_batch(schema, n, rng, values_of):
    """pk strictly increasing from INT64_MIN towards INT64_MAX, sequence numbers with their extremes, every kind;
    values_of(logical type, nullable, n) -> (values, valid mask or None) fills each value column."""
    step = ((1 << 64) - 1) // max(n - 1, 1)
    keys = [I64_MIN + i * step for i in range(n)]
    seq = rng.integers(0, I64_MAX, n, dtype=np.int64, endpoint=True)
    if n > 2:
        seq[rng.integers(0, n)] = 0
        seq[rng.integers(0, n)] = I64_MAX
    kinds = rng.integers(0, 4, n).astype(np.int8)
    types = schema.physical_types()
    cols = [column(types[0], keys), Column(PhysicalType.INT64, seq), Column(PhysicalType.INT8, kinds)]
    for f in schema.value_type.fields:
        vals, valid = values_of(f.type, f.nullable, n)
        cols.append(column(f.physical, vals, valid if f.nullable else None))
    return KeyValueBatch(schema, cols)


def draw(rng, pool, n):
    return [pool[i] for i in rng.integers(0, len(pool), n)]


def mixed_values(rng, nan=True, null_p=0.25):
    """Every row drawn from edges + ordinary values (NaN edges only if `nan`), nullable columns ~25 % NULL."""
    def values_of(logical, nullable, n):
        pool = [v for v in EDGES[logical] if nan or not is_nan_edge(logical, v)] + ORDINARY[logical]
        valid = rng.random(n) >= null_p if nullable else None
        return draw(rng, pool, n), valid
    return values_of


# ---------------------------------------------------------------------------------------------- known answers

def _one_column_schema(logical, nullable=True):
    return KeyValueSchema.of(RowType((DataField("k", "INT", False), DataField("v", logical, nullable))), ["k"])


V = 4                                                           # the value column of _batch


def _batch(logical, values, kinds=None, seqs=None):
    """One value column; None in `values` = NULL."""
    schema = _one_column_schema(logical)
    n = len(values)
    t = schema.physical_types()[V]
    valid = np.array([v is not None for v in values])
    vals = [v if v is not None else (0 if not is_varlen(t) else "") for v in values]
    keys = Column(PhysicalType.INT32, np.arange(n, dtype=np.int32))
    cols = [keys, Column(PhysicalType.INT64, np.asarray(seqs if seqs is not None else np.arange(n) + 100, np.int64)),
            Column(PhysicalType.INT8, np.asarray(kinds if kinds is not None else np.zeros(n), np.int8)), keys,
            column(t, vals, valid)]
    return KeyValueBatch(schema, cols)


def test_writer_rows_round_like_the_encoder():
    assert S.writer_rows() == (32768, 1 << 20)
    assert S.writer_rows(64, 256) == (64, 256)
    assert S.writer_rows(60, 250) == (64, 256)           # pages up to 8 rows, groups up to whole pages
    assert S.writer_rows(1, 1) == (8, 8)
    assert S.writer_rows(100, 1000) == (104, 1040)
    assert S.row_groups(1000, 64, 256) == [(0, 256), (256, 512), (512, 768), (768, 1000)]
    assert S.row_groups(4097) == [(0, 4097)]
    assert S.row_groups(0, 64, 256) == []


def test_integer_footer_bytes_are_sign_extended():
    b = _batch("TINYINT", [5, -128, None, 127])
    st = S.footer_stats(b)[0][V]
    assert st == S.ChunkStats(1, b"\x80\xff\xff\xff", b"\x7f\x00\x00\x00")
    st = S.footer_stats(_batch("SMALLINT", [-32768, 7]))[0][V]
    assert (st.min, st.max) == (b"\x00\x80\xff\xff", b"\x07\x00\x00\x00")
    st = S.footer_stats(_batch("BIGINT", [I64_MAX, I64_MIN, 0]))[0][V]
    assert (st.min, st.max) == (b"\x00" * 7 + b"\x80", b"\xff" * 7 + b"\x7f")
    st = S.footer_stats(_batch("DECIMAL(5,2)", [-99999, 99999]))[0][V]      # unscaled, INT64 physical
    assert (st.min, st.max) == (struct.pack("<q", -99999), struct.pack("<q", 99999))
    assert S.file_stats(_batch("DATE", [None, -719162, 2932896]))[V] == S.FileColStats(-719162, 2932896, 1)


def test_boolean():
    for vals, want in (([1, 1, None], (b"\x01", b"\x01")), ([0, 0], (b"\x00", b"\x00")), ([1, 0, 1], (b"\x00", b"\x01"))):
        st = S.footer_stats(_batch("BOOLEAN", vals))[0][V]
        assert (st.min, st.max) == want
    assert S.file_stats(_batch("BOOLEAN", [1, 0]))[V] == S.FileColStats(False, True, 0)


def test_zero_rule():
    for logical, neg0 in (("DOUBLE", NEG0_F64), ("FLOAT", b"\x00\x00\x00\x80")):
        pos0 = bytes(len(neg0))
        for vals in ([0.0, 0.0], [-0.0, -0.0], [0.0, -0.0, None], [-0.0, 0.0]):
            st = S.footer_stats(_batch(logical, vals))[0][V]
            assert (st.min, st.max) == (neg0, pos0), vals
        st = S.footer_stats(_batch(logical, [0.0, 2.0]))[0][V]          # a zero min is -0.0, a zero max +0.0
        assert st.min == neg0 and S.value_of(PhysicalType.DOUBLE if logical == "DOUBLE" else PhysicalType.FLOAT,
                                              st.max) == 2.0
        st = S.footer_stats(_batch(logical, [-3.0, -0.0]))[0][V]
        assert st.max == pos0
        fs = S.file_stats(_batch(logical, [0.0, 0.0]))[V]
        assert struct.pack("<d", fs.min) == NEG0_F64 and struct.pack("<d", fs.max) == POS0_F64


def test_nan_rule_per_row_group_and_file():
    nan = F64(0x7ff8000000000000)
    vals = [float(i + 1) for i in range(8)] + [2.0, nan, 3.0, None, 4.0, 5.0, 6.0, 7.0]
    b = _batch("DOUBLE", vals)
    groups = S.footer_stats(b, page_rows=8, row_group_rows=8)
    assert len(groups) == 2
    assert groups[0][V] == S.ChunkStats(0, struct.pack("<d", 1.0), struct.pack("<d", 8.0))
    assert groups[1][V] == S.ChunkStats(1, None, None)                  # NaN only in the last row group
    assert S.file_stats(b)[V] == S.FileColStats(None, None, 1)          # ... and the file has no min / max
    # the same NaN in the first row group only, with sign bit and payload
    b = _batch("DOUBLE", [F64(0xfff8000000000001)] + vals[1:8] + [2.0, 3.0])
    groups = S.footer_stats(b, page_rows=8, row_group_rows=8)
    assert not groups[0][V].has_min_max and groups[1][V].has_min_max
    assert S.file_stats(b)[V].min is None
    # a NaN under a NULL is not a value
    b = _batch("FLOAT", [1.0, 2.0])
    b.columns[V] = column(PhysicalType.FLOAT, [F32(0x7fc00000), 2.0], np.array([False, True]))
    assert S.file_stats(b)[V] == S.FileColStats(2.0, 2.0, 1)
    assert S.file_stats(_batch("FLOAT", [F32(0x7fc00000)]))[V] == S.FileColStats(None, None, 0)


def test_all_null_and_strings():
    assert S.footer_stats(_batch("BIGINT", [None] * 5))[0][V] == S.ChunkStats(5, None, None)
    assert S.file_stats(_batch("DOUBLE", [None] * 3))[V] == S.FileColStats(None, None, 3)
    assert S.footer_stats(_batch("STRING", ["a", None, "b"]))[0][V] == S.ChunkStats(1, None, None)
    assert S.file_stats(_batch("STRING", ["a", None, "b"]))[V] == S.FileColStats(None, None, 1)


def test_slices_see_only_their_rows():
    b = _batch("INT", [-7, 1, 2, 3, 4, 5, 6, 7] + [10, 11, None, 13, 14] + [99, 100])
    assert S.file_stats(b, 8, 5)[V] == S.FileColStats(10, 14, 1)
    assert [g[V] for g in S.footer_stats(b, 8, 5, page_rows=8, row_group_rows=8)] == \
        [S.ChunkStats(1, struct.pack("<i", 10), struct.pack("<i", 14))]
    m = S.data_file_meta(b, 8, 5)
    assert (m.row_count, m.min_key, m.max_key, m.min_sequence_number, m.max_sequence_number) == (5, 8, 12, 108, 112)


def test_data_file_meta():
    b = _batch("INT", [1, 2, 3, 4, 5], kinds=[0, 1, 2, 3, 1], seqs=[9, I64_MAX, 0, 5, 7])
    assert S.data_file_meta(b) == S.FileMeta(5, 0, I64_MAX, 3, 0, 4)
    assert S.data_file_meta(b, 0, 0) == S.FileMeta(0, None, None, 0, None, None)
    vt = RowType((DataField("a", "INT", False), DataField("b", "STRING", False), DataField("v", "INT", True)))
    schema = KeyValueSchema.of(vt, ["a", "b"])
    b = KeyValueBatch.from_rows(schema, [(1, "x", 0, 0, 1, "x", 5), (2, "y", 1, 2, 2, "y", 6)])
    m = S.data_file_meta(b)
    assert (m.min_key, m.max_key, m.delete_row_count) == ((1, "x"), (2, "y"), 0)


def test_java_compare_is_double_compare():
    jc = S.java_compare
    assert jc(-0.0, 0.0) == -1 and jc(0.0, -0.0) == 1 and jc(-0.0, -0.0) == 0
    nan, nan_neg, nan_pay = float("nan"), float(F64(0xfff8000000000000)), float(F64(0x7ff4000000000123))
    assert jc(nan, np.inf) == 1 and jc(np.inf, nan) == -1
    assert jc(nan, nan_neg) == 0 and jc(nan_pay, nan) == 0            # every NaN is the same NaN
    assert jc(nan_neg, -np.inf) == 1                                  # the sign bit of a NaN does not count
    assert jc(-np.inf, -1.7976931348623157e308) == -1 and jc(5e-324, 0.0) == 1 and jc(-5e-324, -0.0) == -1
    assert jc(1, 2) == -1 and jc(I64_MAX, I64_MIN) == 1 and jc(3, 3) == 0


def test_soundness_check_catches_a_positive_zero_min():
    T = PhysicalType.DOUBLE
    assert S.unsound(T, 0.0, 0.0, np.array([-0.0, 0.0])) == [-0.0]
    assert S.unsound(T, -0.0, 0.0, np.array([-0.0, 0.0])) == []
    assert S.unsound(T, 1.0, 5.0, np.array([1.0, np.nan, 5.0]))       # a NaN above every finite max
    assert S.unsound(T, None, None, np.array([np.nan])) == []
    assert S.unsound(PhysicalType.INT64, -1, 4, np.array([-1, 5])) == [5]


# ---------------------------------------------------------------------------------------------- against pyarrow

def _pyarrow_row_groups(batch, path, group):
    pq.write_table(to_arrow(batch), path, row_group_size=group, use_dictionary=False, compression="none",
                   write_statistics=True)
    md = pq.ParquetFile(path).metadata
    out = []
    for g in range(md.num_row_groups):
        row = []
        for c, t in enumerate(batch.schema.physical_types()):
            cs = md.row_group(g).column(c).statistics
            if is_varlen(t):
                row.append(None)
            elif cs.has_min_max:
                row.append(S.ChunkStats(cs.null_count, S.footer_bytes(t, cs.min), S.footer_bytes(t, cs.max)))
            else:
                row.append(S.ChunkStats(cs.null_count, None, None))
        out.append(row)
    return out


def _zeros_and_infinities(rng):
    """NaN-free pools, zeros and infinities frequent: the rules pyarrow's writer shares with the model."""
    def values_of(logical, nullable, n):
        pool = [v for v in EDGES[logical] if not is_nan_edge(logical, v)]
        if logical in ("FLOAT", "DOUBLE"):
            mode = rng.integers(0, 4)
            pool = [[0.0], [-0.0], [0.0, -0.0], pool + ORDINARY[logical]][mode]
        valid = rng.random(n) >= 0.3 if nullable else None
        return draw(rng, pool, n), valid
    return values_of


@pytest.mark.parametrize("n,seed", [(1, 0), (8, 1), (300, 2), (1000, 3), (1000, 4), (2048, 5)])
def test_model_agrees_with_pyarrow(tmp_path, n, seed):
    schema = stats_schema()
    rng = np.random.default_rng(seed)
    batch = make_batch(schema, n, rng, mixed_values(rng, nan=False) if seed % 2 else _zeros_and_infinities(rng))
    want = S.footer_stats(batch, page_rows=64, row_group_rows=256)
    got = _pyarrow_row_groups(batch, str(tmp_path / "pa.parquet"), 256)
    assert len(got) == len(want)
    types = schema.physical_types()
    for g, (gw, gg) in enumerate(zip(want, got)):
        for c, (w, x) in enumerate(zip(gw, gg)):
            if not is_varlen(types[c]):
                assert w == x, f"row group {g} column {schema.file_fields()[c].name}"


def test_model_agrees_with_pyarrow_on_constant_zero_chunks(tmp_path):
    """Row groups of only +0.0, only -0.0, and both, for FLOAT and DOUBLE."""
    schema = stats_schema()
    zeros = [[0.0] * 256, [-0.0] * 256, [0.0, -0.0] * 128]
    def values_of(logical, nullable, n):
        if logical in ("FLOAT", "DOUBLE"):
            return sum(zeros, []), None
        return draw(np.random.default_rng(1), ORDINARY[logical], n), None
    batch = make_batch(schema, 768, np.random.default_rng(0), values_of)
    want = S.footer_stats(batch, page_rows=64, row_group_rows=256)
    got = _pyarrow_row_groups(batch, str(tmp_path / "z.parquet"), 256)
    f = schema.physical_types().index(PhysicalType.DOUBLE)
    for g in range(3):
        assert want[g][f] == got[g][f] == S.ChunkStats(0, NEG0_F64, POS0_F64)
        for c, t in enumerate(schema.physical_types()):
            if t in (PhysicalType.FLOAT, PhysicalType.DOUBLE):
                assert want[g][c] == got[g][c]
