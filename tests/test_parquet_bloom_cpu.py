"""Parquet split-block bloom filters without a device: the model in parquet_bloom_reference.py against pyarrow's
writer bit for bit, the host build of sbbf_device.cuh (the source k_pw_sbbf compiles, tests/native/
parquet_bloom_host_check.cc, under AddressSanitizer and UBSan) against the model, and the rewriter's reading of the
'parquet.bloom.filter.*' table options."""
import io
import os
import random
import struct
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest
import xxhash

import parquet_bloom_reference as R
from paimon_b200 import _native as N
from paimon_b200.compact_rewriter import (KeyValueDataFileWriter, MergeTreeCompactRewriter, file_column_names,
                                          parquet_bloom_for_level)
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.types import DataField, KeyValueSchema, RowType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (ndv, fpp) pairs whose filter size parquet-mr's sizing and Arrow's agree on
AGREED_SIZES = [((1000, 0.01), 2048), ((10, 0.1), 32), ((100000, 0.05), 131072), ((5000, 0.01), 8192), ((1, 0.5), 32)]


@pytest.fixture(scope="module")
def host_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sbbf") / "parquet_bloom_host_check")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I" + os.path.join(ROOT, "paimon_b200", "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", "native", "parquet_bloom_host_check.cc")])

    def run(lines):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        p = subprocess.run([exe], input="".join(l + "\n" for l in lines), capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        out = p.stdout.splitlines()
        assert len(out) == len(lines)
        return out
    return run


def _pyarrow_file(table, ndv, fpp, row_group_size=None):
    sink = io.BytesIO()
    pq.write_table(table, sink, use_dictionary=False, row_group_size=row_group_size,
                   bloom_filter_options={c: {"ndv": ndv, "fpp": fpp} for c in table.column_names})
    return sink.getvalue()


def _edge_table(n, seed):
    rng = np.random.default_rng(seed)
    valid = rng.random(n) > 0.2
    strs = [None if not v else "".join(chr(0x61 + int(x) % 26) for x in rng.integers(0, 26, int(rng.choice([0, 1, 7, 31, 32, 33, 100]))))
            for v in valid]
    f32 = rng.normal(size=n).astype(np.float32)
    f32[:4] = [np.nan, -0.0, 0.0, np.inf]
    f64 = rng.normal(size=n)
    f64[:4] = [np.nan, -0.0, 0.0, -np.inf]
    mask = ~valid
    mask[:4] = False
    return pa.table({
        "i8": pa.array(rng.integers(-128, 128, n).astype(np.int8), mask=mask),
        "i16": pa.array(rng.integers(-2 ** 15, 2 ** 15, n).astype(np.int16), mask=mask),
        "i32": pa.array(rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32), mask=mask),
        "i64": pa.array(rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64), mask=mask),
        "date": pa.array(rng.integers(-20000, 20000, n).astype(np.int32), mask=mask).cast(pa.date32()),
        "f32": pa.array(f32, mask=mask),
        "f64": pa.array(f64, mask=mask),
        "s": pa.array(strs, pa.string()),
        "b": pa.array([None if s is None else s.encode() + b"\xff\x00" for s in strs], pa.binary()),
    })


KIND = {"i8": "int32", "i16": "int32", "i32": "int32", "i64": "int64", "date": "int32", "f32": "float", "f64": "double",
        "s": "bytes", "b": "bytes"}


def _values(col):
    """The values of a pyarrow column as the model hashes them: FLOAT / DOUBLE by their bits, DATE as days."""
    if pa.types.is_date32(col.type):
        col = col.cast(pa.int32())
    if pa.types.is_float32(col.type) or pa.types.is_float64(col.type):
        bits = np.asarray(col.fill_null(0).to_numpy(zero_copy_only=False)).view(
            np.uint32 if pa.types.is_float32(col.type) else np.uint64)
        return [None if v is None else int(b) for v, b in zip(col.to_pylist(), bits)]
    return col.to_pylist()


@pytest.mark.parametrize("ndv_fpp,size", AGREED_SIZES[:3])
def test_model_equals_pyarrow_bit_for_bit(ndv_fpp, size):
    ndv, fpp = ndv_fpp
    table = _edge_table(3000, seed=ndv)
    data = _pyarrow_file(table, ndv, fpp, row_group_size=1100)         # three row groups, the last one short
    filters = R.file_filters(data)
    assert len(filters) == 3
    r0 = 0
    for g, row in enumerate(filters):
        n = pq.ParquetFile(io.BytesIO(data)).metadata.row_group(g).num_rows
        for c, name in enumerate(table.column_names):
            f = row[c]
            assert f is not None and f["header"][1] == size == R.num_bytes(ndv, fpp), (name, g)
            vals = _values(table.column(name).slice(r0, n))
            assert f["bitset"] == R.build(KIND[name], vals, size), (name, g)
            assert all(R.contains(f["bitset"], KIND[name], v) for v in vals if v is not None)
        r0 += n


def test_float_zeros_and_nan_are_their_own_bits():
    # -0.0 and +0.0, and two NaN payloads, hash differently: the bits are hashed as they are
    assert R.hash_value("float", 0x80000000) != R.hash_value("float", 0)
    assert R.hash_value("double", 0x7FF8000000000000) != R.hash_value("double", 0x7FF8000000000001)
    assert R.hash_value("float", -0.0) == R.hash_value("float", 0x80000000)
    assert R.hash_value("bytes", "") == xxhash.xxh64_intdigest(b"")


@pytest.mark.parametrize("ndv_fpp,size", AGREED_SIZES)
def test_sizing_where_parquet_mr_and_arrow_agree(ndv_fpp, size):
    ndv, fpp = ndv_fpp
    assert R.num_bytes(ndv, fpp) == size
    data = _pyarrow_file(pa.table({"a": pa.array(np.arange(10, dtype=np.int64))}), ndv, fpp)
    assert R.file_filters(data)[0][0]["header"][1] == size


def test_sizing_model():
    assert R.num_bytes(0) == R.num_bytes(0, 0.5) == 1 << 20            # no ndv: parquet-mr's default maximum
    assert R.num_bytes(10 ** 6, 0.01) == 1 << 20                       # capped where Arrow would write 2 MiB
    assert R.num_bytes(10 ** 12, 0.01) == 1 << 20                      # past the spec's bound
    assert R.num_bytes(1, 0.999999) == 32
    sizes = {R.num_bytes(n, f) for n in (1, 10, 1000, 10 ** 5, 10 ** 7) for f in (0.5, 0.1, 0.01, 1e-6)}
    assert all(s & (s - 1) == 0 and 32 <= s <= 1 << 20 for s in sizes)


def test_device_sizing_and_hashes(host_check):
    ndvs = [1, 2, 10, 99, 1000, 12345, 10 ** 5, 10 ** 6, 10 ** 9, 2 ** 40]
    fpps = [0.5, 0.1, 0.05, 0.01, 0.001, 1e-6, 1e-12, 0.999999]
    cases = [(0, 0.01)] + [(n, f) for n in ndvs for f in fpps]
    assert host_check([f"s {n} {f!r}" for n, f in cases]) == [str(R.num_bytes(n, f)) for n, f in cases]
    rng = random.Random(3)
    v32 = [0, 1, 0xFFFFFFFF, 0x80000000, 0x7FC00000] + [rng.getrandbits(32) for _ in range(200)]
    v64 = [0, 1, 2 ** 64 - 1, 2 ** 63, 0x7FF8000000000000] + [rng.getrandbits(64) for _ in range(200)]
    out = host_check([f"4 {v}" for v in v32] + [f"8 {v}" for v in v64])
    want = [xxhash.xxh64_intdigest(struct.pack("<I", v)) for v in v32] + \
           [xxhash.xxh64_intdigest(struct.pack("<Q", v)) for v in v64]
    assert out == [f"{w} {w}" for w in want]


def test_device_filter_bits(host_check):
    rng = random.Random(5)
    lines, want = [], []
    for size in (32, 64, 2048, 8192):
        for n in (0, 1, 5, 100, 2000):
            vals = [bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 4, 8, 31, 32, 33, 70]))) for _ in range(n)]
            lines.append(f"f {size} " + " ".join(v.hex() or "-" for v in vals))
            want.append(R.build("bytes", vals, size).hex())
    assert host_check(lines) == want


# ---- the rewriter's reading of the table options

def bloom_schema():
    fields = [DataField("pk", "BIGINT", False), DataField("a", "INT", True), DataField("flag", "BOOLEAN", True),
              DataField("s", "STRING", True), DataField("d", "DOUBLE", True)]
    return KeyValueSchema.of(RowType(tuple(fields)), ["pk"])


def test_option_parsing():
    schema = bloom_schema()
    names = file_column_names(schema)
    assert names == ["_KEY_pk", "_SEQUENCE_NUMBER", "_VALUE_KIND", "pk", "a", "flag", "s", "d"]
    col = {n: i for i, n in enumerate(names)}
    assert parquet_bloom_for_level(schema, None) == []
    assert parquet_bloom_for_level(schema, {"parquet.bloom.filter.enabled": "false"}) == []
    # the global flag: every file column, key and system columns included, BOOLEAN left out
    got = parquet_bloom_for_level(schema, {"parquet.bloom.filter.enabled": "TRUE"})
    assert got == [(col[n], 0, 0.01) for n in names if n != "flag"]
    # overrides both ways, an unknown '#col' ignored, ndv and fpp per column
    got = parquet_bloom_for_level(schema, {
        "parquet.bloom.filter.enabled": "true", "parquet.bloom.filter.enabled#a": "false",
        "parquet.bloom.filter.enabled#nope": "true", "parquet.bloom.filter.expected.ndv#s": "5000",
        "parquet.bloom.filter.fpp#s": "0.05", "parquet.bloom.filter.fpp#_KEY_pk": "0.1",
        "parquet.bloom.filter.expected.ndv#nope": "7"})
    assert got == [(col["_KEY_pk"], 0, 0.1), (col["_SEQUENCE_NUMBER"], 0, 0.01), (col["_VALUE_KIND"], 0, 0.01),
                   (col["pk"], 0, 0.01), (col["s"], 5000, 0.05), (col["d"], 0, 0.01)]
    got = parquet_bloom_for_level(schema, {"parquet.bloom.filter.enabled#_KEY_pk": "true",
                                           "parquet.bloom.filter.enabled#d": "true",
                                           "parquet.bloom.filter.enabled#flag": "true",
                                           "parquet.bloom.filter.expected.ndv#d": "100"})
    assert got == [(col["_KEY_pk"], 0, 0.01), (col["d"], 100, 0.01)]


BAD_OPTIONS = [
    {"parquet.bloom.filter.expected.ndv#a": "many"},
    {"parquet.bloom.filter.expected.ndv#a": "0"},
    {"parquet.bloom.filter.expected.ndv#a": "-5"},
    {"parquet.bloom.filter.fpp#a": "often"},
    {"parquet.bloom.filter.fpp#a": "0"},
    {"parquet.bloom.filter.fpp#a": "1.0"},
    {"parquet.bloom.filter.fpp#nope": "2"},
]


@pytest.mark.parametrize("options", BAD_OPTIONS)
def test_bad_ndv_or_fpp_is_refused_before_any_device_work(tmp_path, options):
    schema = bloom_schema()
    options = dict(options, **{"parquet.bloom.filter.enabled": "true", "file.format": "parquet"})
    with pytest.raises(N.PaimonGpuError, match="parquet encode: option parquet.bloom.filter"):
        parquet_bloom_for_level(schema, options)
    rewriter = MergeTreeCompactRewriter(schema, DeduplicateMergeFunction.factory(), str(tmp_path), options=options)
    with pytest.raises(N.PaimonGpuError, match="parquet encode: option parquet.bloom.filter"):
        rewriter.rewrite_compaction(1, False, [])
    assert os.listdir(tmp_path) == []


def test_orc_levels_ignore_the_parquet_options(tmp_path):
    # an ORC output level never reads them, so even a malformed one does not stop it
    schema = bloom_schema()
    options = {"file.format": "orc", "parquet.bloom.filter.enabled": "true", "parquet.bloom.filter.fpp#a": "2"}
    rewriter = MergeTreeCompactRewriter(schema, DeduplicateMergeFunction.factory(), str(tmp_path), options=options)
    assert rewriter.rewrite_compaction(1, False, []).after == []


def test_writer_builds_the_bloom_options():
    w = KeyValueDataFileWriter(bloom_schema(), "/nonexistent/f.parquet", 1, parquet_bloom=[(4, 1000, 0.05), (6, 0, 0.01)])
    b = w.parquet_bloom
    assert b.n_columns == 2
    assert [(b.columns[i].column, b.columns[i].ndv, b.columns[i].fpp) for i in range(2)] == [(4, 1000, 0.05), (6, 0, 0.01)]
    assert KeyValueDataFileWriter(bloom_schema(), "/nonexistent/f.parquet", 1).parquet_bloom.n_columns == 0
