"""The ORC row index model (tests/orc_index_reference.py) against files pyarrow.orc writes through the Apache ORC C++
writer with row_index_stride= and bloom_filter_columns=: the BLOOM_FILTER_UTF8 bit sets bit for bit, the row group
statistics on the fields both writers carry, and the number of positions per entry for each column kind, with and
without nulls, uncompressed and ZSTD.  Also: k_oe_bloom compiles for sm_90a without spills, the ctypes mirror of
pg_orc_index_options, and the writer's refusals of index options, raised before any device work."""
import io
import os
import re
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.orc as orc
import pytest

import orc_index_reference as X
import orc_stats_reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, arrow type, ORC kind, values of n rows)
def _columns(rng, n):
    words = ["", "a", "paimon", "é€", "x" * 17, "orc-index", "0123456789abcdef"]
    return [
        ("i8", pa.int8(), 1, rng.integers(-128, 128, n).astype(np.int8)),
        ("i16", pa.int16(), 2, rng.integers(-2 ** 15, 2 ** 15, n).astype(np.int16)),
        ("i32", pa.int32(), 3, rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32)),
        ("i64", pa.int64(), 4, rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64)),
        ("f32", pa.float32(), 5, rng.uniform(-1e3, 1e3, n).astype(np.float32)),
        ("f64", pa.float64(), 6, rng.standard_normal(n) * 1e6),
        ("s", pa.string(), 7, [rng.choice(words) + str(int(rng.integers(0, 50))) for _ in range(n)]),
        ("bin", pa.binary(), 8, [bytes(rng.integers(0, 256, int(rng.integers(0, 12))).astype(np.uint8)) for _ in range(n)]),
        ("dt", pa.date32(), 15, rng.integers(-10000, 30000, n).astype(np.int32)),
    ]


def _table(n, null_p, seed):
    rng = np.random.default_rng(seed)
    cols, model = {}, []
    for name, t, kind, vals in _columns(rng, n):
        valid = rng.random(n) >= null_p
        py = vals.tolist() if isinstance(vals, np.ndarray) else vals
        arr = pa.array([v if ok else None for v, ok in zip(py, valid)], pa.int32() if t == pa.date32() else t)
        cols[name] = arr.cast(t) if t == pa.date32() else arr
        mv = [v.encode() if isinstance(v, str) else v for v in vals] if isinstance(vals, list) else vals
        model.append((kind, mv, valid, 0))
    return pa.table(cols), model


def _write(table, stride, compression="uncompressed", bloom=(), fpp=0.05):
    buf = io.BytesIO()
    orc.write_table(table, buf, compression=compression, row_index_stride=stride, bloom_filter_columns=list(bloom),
                    bloom_filter_fpp=fpp)
    return buf.getvalue()


@pytest.mark.parametrize("fpp", [0.01, 0.05])
@pytest.mark.parametrize("null_p", [0.0, 0.3])
def test_filters_equal_pyarrow(fpp, null_p):
    n, stride = 3500, 1000                                   # 3 full row groups and a short one
    table, model = _table(n, null_p, seed=int(fpp * 100) + int(null_p * 10))
    blob = _write(table, stride, bloom=range(1, len(model) + 1), fpp=fpp)
    got_stride, stripes = X.read_file(blob)
    assert got_stride == stride and len(stripes) == 1
    bits, k = X.sizing(stride, fpp)
    assert bits % 64 == 0 and bits > -stride * np.log(fpp) / np.log(2) ** 2
    for c, (kind, vals, valid, _) in enumerate(model):
        filters = stripes[0].bloom[c + 1]
        assert len(filters) == 4
        for g, (r0, r1) in enumerate(X.row_groups(n, n, stride)[0]):
            want = X.bloom_bitset(X.hashes(kind, vals[r0:r1], valid[r0:r1]), bits, k)
            if kind == 1:
                # The ORC C++ writer's TINYINT filters are not orc-core's: a filter of 1000 copies of 1 also holds the
                # bits of 0x0101010101010101, and negative values are not hashed sign-extended.  orc-core's
                # ByteTreeWriter adds the sign-extended value, which the model follows; only the sizing is compared.
                assert filters[g][0] == k and len(filters[g][1]) == len(want), g
            else:
                assert filters[g] == (k, want), (kind, g)


def test_sizing_matches_pyarrow_and_orc_core():
    assert X.sizing(10000, 0.05) == (62400, 4)
    assert X.sizing(10000, 0.01) == (95872, 7)
    # the hash of a value of every length 0..20 against a filter pyarrow wrote of that one value
    values = ["ab" * (i // 2) + "c" * (i % 2) for i in range(21)]
    for v in values:
        blob = _write(pa.table({"s": pa.array([v] * 1000)}), 1000, bloom=[1], fpp=0.05)
        [(k, bitset)] = X.read_file(blob)[1][0].bloom[1]
        assert bitset == X.bloom_bitset(np.array([X.murmur3_hash64(v.encode())], np.uint64), *X.sizing(1000, 0.05))


def test_special_doubles_hash_like_pyarrow():
    """NaN, both zeros and infinities: DOUBLE by its bits with NaN canonical, FLOAT widened first"""
    vals = [float("nan"), 0.0, -0.0, float("inf"), -float("inf"), 1.5, -2.25] * 150
    table = pa.table({"d": pa.array(vals, pa.float64()), "f": pa.array(vals, pa.float32())})
    blob = _write(table, 1000, bloom=[1, 2], fpp=0.01)
    st = X.read_file(blob)[1][0]
    for c, kind in ((1, 6), (2, 5)):
        v = np.asarray(vals, np.float64 if kind == 6 else np.float32)
        for g, (r0, r1) in enumerate(X.row_groups(len(vals), len(vals), 1000)[0]):
            want = X.bloom_bitset(X.hashes(kind, v[r0:r1], np.ones(r1 - r0, bool)), *X.sizing(1000, 0.01))
            assert st.bloom[c][g][1] == want, (kind, g)


@pytest.mark.parametrize("null_p", [0.0, 0.3])
def test_statistics_equal_pyarrow_on_shared_fields(null_p):
    n, stride = 2600, 1000
    table, model = _table(n, null_p, seed=3)
    _, stripes = X.read_file(_write(table, stride))
    want = X.expected_entries(model, n, n, stride)[0]
    for c, entries in enumerate(want):
        got = stripes[0].index[c]
        assert len(got) == len(entries)
        for g, (w, (_, s)) in enumerate(zip(entries, got)):
            shared = {k: s[k] for k in w if k in s}
            assert ref.same(shared, w), (c, g, s, w)


@pytest.mark.parametrize("compression", ["uncompressed", "zstd"])
def test_position_counts_equal_pyarrow(compression):
    n, stride = 2500, 1000
    for null_p in (0.0, 0.3):
        table, model = _table(n, null_p, seed=9)
        dec = pa.array([None if null_p and i % 3 == 0 else i * 7 for i in range(n)], pa.decimal128(15, 4))
        bools = pa.array([None if null_p and i % 5 == 0 else i % 3 == 0 for i in range(n)], pa.bool_())
        table = table.append_column("dec", dec).append_column("b", bools)
        kinds = [m[0] for m in model] + [X.DECIMAL, X.BOOLEAN]
        _, stripes = X.read_file(_write(table, stride, compression), decompress=_zstd_decompress)
        for c, kind in enumerate(kinds):
            has_present = (c + 1, X.PRESENT) in stripes[0].streams
            assert has_present == (null_p > 0)
            for positions, _ in stripes[0].index[c + 1]:
                assert len(positions) == X.position_count(kind, has_present, compression == "zstd"), (kind, null_p)
        assert all(not p for p, _ in stripes[0].index[0])         # the root has none


def _zstd_decompress(frame):
    import codec_filter
    global _CODEC
    if "_CODEC" not in globals():
        import tempfile
        _CODEC = codec_filter.build(tempfile.mkdtemp())
    from codec_corpora import ZSTD
    [(r, out)] = _CODEC([(ZSTD, frame, 1 << 20)])
    assert r >= 0
    return out


def test_bloom_kernel_compiles_without_spills():
    res = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                          "-Xptxas", "-v", "-I" + os.path.join(ROOT, "include"),
                          "-I" + os.path.join(ROOT, "paimon_b200", "csrc"), "-x", "cu", "-c", "-o", os.devnull,
                          os.path.join(ROOT, "paimon_b200", "csrc", "orc_encode.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    at = next(i for i, l in enumerate(lines) if "Function properties for" in l and "k_oe_bloom" in l)
    assert re.search(r"0 bytes spill stores, 0 bytes spill loads", lines[at + 1]), lines[at:at + 3]


def test_index_options_struct_and_refusals():
    from paimon_b200 import _native as N
    from paimon_b200.compact_rewriter import KeyValueDataFileWriter, orc_index_for_level
    from paimon_b200.types import DataField, KeyValueSchema, RowType
    assert [(f, t) for f, t in N.PgOrcIndexOptions._fields_] == [
        ("row_index_stride", N.C.c_int64), ("n_bloom_columns", N.C.c_int32),
        ("bloom_columns", N.C.POINTER(N.C.c_int32)), ("bloom_fpp", N.C.c_double)]
    hdr = open(os.path.join(ROOT, "include", "paimon_gpu.h")).read()
    body = hdr[hdr.index("int64_t row_index_stride;"):hdr.index("} pg_orc_index_options;")]
    assert re.findall(r"\b(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S)) == ["row_index_stride", "n_bloom_columns", "bloom_columns", "bloom_fpp"]
    schema = KeyValueSchema.of(RowType((DataField("pk", "INT", False), DataField("b", "BOOLEAN", True),
                                        DataField("dec", "DECIMAL(10,2)", True), DataField("s", "STRING", True))), ["pk"])

    def writer(**kw):
        return KeyValueDataFileWriter(schema, os.devnull, 0, file_format="orc", **kw)
    assert writer(row_index_stride=10000, bloom_filter_columns=["s", "pk"]).orc_index.n_bloom_columns == 2
    assert list(writer(row_index_stride=1000, bloom_filter_columns=["s"]).orc_index.bloom_columns[:1]) == [6]
    assert writer().orc_index.row_index_stride == 0
    for kw in (dict(row_index_stride=999), dict(row_index_stride=-8), dict(bloom_filter_columns=["s"]),
               dict(row_index_stride=1000, bloom_filter_columns=["s"], bloom_filter_fpp=1.0),
               dict(row_index_stride=1000, bloom_filter_columns=["s", "s"]),
               dict(row_index_stride=1000, bloom_filter_columns=["nope"])):
        with pytest.raises(N.PaimonGpuError) as e:
            writer(**kw)
        assert e.value.status == 1, kw
    for kw in (dict(row_index_stride=1004), dict(row_index_stride=1000, bloom_filter_columns=["b"]),
               dict(row_index_stride=1000, bloom_filter_columns=["dec"]),
               dict(row_index_stride=10 ** 6, bloom_filter_columns=["s"], bloom_filter_fpp=1e-6)):
        with pytest.raises(N.UnsupportedOnDevice):
            writer(**kw)
    # Parquet files ignore the ORC options
    KeyValueDataFileWriter(schema, os.devnull, 0, row_index_stride=3)
    assert orc_index_for_level({}) == dict(row_index_stride=10000, bloom_filter_columns=(), bloom_filter_fpp=0.01)
    assert orc_index_for_level({"orc.create.index": "false", "orc.bloom.filter.columns": "s"}) == \
        dict(row_index_stride=0, bloom_filter_columns=())
    assert orc_index_for_level({"orc.row.index.stride": "2000", "orc.bloom.filter.columns": "s, pk",
                                "orc.bloom.filter.fpp": "0.05"}) == \
        dict(row_index_stride=2000, bloom_filter_columns=("s", "pk"), bloom_filter_fpp=0.05)
