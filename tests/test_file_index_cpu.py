"""The bloom-filter file index without a device: the hashes, bit positions and sizing of xxhash64_device.cuh (compiled
for the host under AddressSanitizer and UBSan from the same source k_bloom_build uses, tests/native/
file_index_host_check.cc), the host-only size query of the C ABI, and file_index.py (options, MemorySize, the
FileIndexFormat container and its HashMap column order, the embedded-or-side-file choice, the refusals), all against
the independent model in file_index_reference.py."""
import ctypes as C
import os
import random
import struct
import subprocess

import numpy as np
import pytest
import xxhash

import file_index_reference as R
from paimon_b200 import _native as N
from paimon_b200.compact_rewriter import KeyValueDataFileWriter, MergeTreeCompactRewriter
from paimon_b200.file_index import (DataFileIndexWriter, FileIndexOptions, parse_memory_size, serialize_file_index,
                                    write_utf)
from paimon_b200.format import LocalFileIO
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.types import DataField, KeyValueSchema, RowType

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host_check(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("fi") / "file_index_host_check")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I" + os.path.join(ROOT, "paimon_b200", "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", "native", "file_index_host_check.cc")])

    def run(lines):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        p = subprocess.run([exe], input="".join(l + "\n" for l in lines), capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        out = p.stdout.splitlines()
        assert len(out) == len(lines)
        return out
    return run


def test_xxh64_model_matches_xxhash_and_the_published_vectors():
    # the specification's vectors for seed 0: "", "a", "abc"
    assert R.xxh64(b"") == 0xEF46DB3751D8E999
    assert R.xxh64(b"a") == 0xD24EC4F1A98C6E5B
    assert R.xxh64(b"abc") == 0x44BC2CF5AD770999
    rng = random.Random(3)
    for n in list(range(0, 80)) + [127, 128, 129, 255, 256, 1000, 4099]:
        data = bytes(rng.randrange(256) for _ in range(n))
        assert R.xxh64(data) == xxhash.xxh64(data, seed=0).intdigest(), n


def test_device_xxh64_every_length_and_alignment(host_check):
    rng = random.Random(11)
    data = bytes(rng.randrange(256) for _ in range(300))
    lines, want = [], []
    for n in range(301):
        for align in range(16):
            lines.append(f"x {align} {data[:n].hex()}")
            want.append(str(R.xxh64(data[:n])))
    assert host_check(lines) == want


INT_EDGES = sorted({v for b in (8, 16, 32, 64) for v in (-(1 << (b - 1)), (1 << (b - 1)) - 1)} | {-1, 0, 1, 42})
FLOAT_BITS = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7FC00001, 0xFFC00000, 0x7F800001,
              0xFFFFFFFF, 0x00000001, 0x3F800000, 0xBF800000, 0x7F7FFFFF]
DOUBLE_BITS = [0, 1 << 63, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0x7FF8000000000001,
               0xFFF8000000000000, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF, 1, 0x3FF0000000000000,
               0xBFF0000000000000, 0x7FEFFFFFFFFFFFFF]


def test_device_integer_and_float_hashes(host_check):
    lines = [f"w {v}" for v in INT_EDGES] + [f"f {b}" for b in FLOAT_BITS] + [f"d {b}" for b in DOUBLE_BITS]
    want = ([R.get_long_hash(v) for v in INT_EDGES] + [R.fast_hash("FLOAT", ("bits", b)) for b in FLOAT_BITS]
            + [R.fast_hash("DOUBLE", ("bits", b)) for b in DOUBLE_BITS])
    assert host_check(lines) == [str(w) for w in want]
    # every NaN payload folds to the canonical NaN: one hash for all of them
    nan_f = {R.fast_hash("FLOAT", ("bits", b)) for b in (0x7FC00000, 0x7FC00001, 0xFFC00000, 0x7F800001, 0xFFFFFFFF)}
    assert len(nan_f) == 1


def test_device_sizing_and_bit_positions(host_check):
    cases = [(i, f) for i in (1, 7, 100, 10 ** 6, 10 ** 9) for f in (0.5, 0.1, 0.01, 1e-6)]
    got = host_check([f"s {i} {f!r}" for i, f in cases])
    for (i, f), g in zip(cases, got):
        want = R.sizing(i, f)
        assert g == ("refused" if want is None else f"{want[0]} {want[1]}"), (i, f)
    assert R.sizing(10 ** 6, 0.1) == (4792536, 3) and R.sizing(100, 0.1) == (480, 3)
    assert R.sizing(10 ** 9, 0.1) is None                      # Java's int overflows: no bit set can be allocated
    rng = random.Random(5)
    hashes = [rng.randrange(-(1 << 63), 1 << 63) for _ in range(300)] + [0, -1, (1 << 63) - 1, -(1 << 63)]
    lines, want = [], []
    for h in hashes:
        for k, bits in ((3, 480), (1, 8), (7, 4792536), (20, 2147483640)):
            lines.append(f"b {h} {k} {bits}")
            want.append(" ".join(map(str, R.positions(h, k, bits))))
    assert host_check(lines) == want


def test_size_query_of_the_c_abi_needs_no_device():
    lib = N.load()
    for items in (1, 7, 100, 10 ** 6, 10 ** 9):
        for fpp in (0.5, 0.1, 0.01, 1e-6):
            size, k = C.c_int64(0), C.c_int32(0)
            st = lib.pg_bloom_filter_size(items, fpp, C.byref(size), C.byref(k))
            want = R.sizing(items, fpp)
            if want is None:
                assert st == 1 and b"2^31" in lib.pg_last_error()
            else:
                assert st == 0 and (size.value, k.value) == (4 + want[0] // 8, want[1]), (items, fpp)
    for items, fpp in ((0, 0.1), (-5, 0.1), (100, 0.0), (100, 1.0), (100, -0.5), (100, 2.0), (100, float("nan"))):
        assert lib.pg_bloom_filter_size(items, fpp, None, None) == 1, (items, fpp)
        # the build checks its specs before it looks at the handle or the device
        spec = N.PgBloomFilterSpec(3, items, fpp)
        buf = (C.c_uint8 * 8)()
        outs = (C.c_void_p * 1)(C.addressof(buf))
        caps = (C.c_int64 * 1)(8)
        assert lib.pg_bloom_filter_build(12345, 0, -1, 1, C.byref(spec), outs, caps) == 1
        assert b"pg_init" not in lib.pg_last_error()


def test_memory_size():
    assert parse_memory_size("500 B") == 500
    assert parse_memory_size("0") == 0
    assert parse_memory_size(" 12 ") == 12
    for unit, mult in (("b", 1), ("k", 1 << 10), ("kb", 1 << 10), ("m", 1 << 20), ("mb", 1 << 20), ("g", 1 << 30),
                       ("gb", 1 << 30), ("t", 1 << 40), ("tb", 1 << 40)):
        assert parse_memory_size(f"3{unit}") == 3 * mult
        assert parse_memory_size(f"3 {unit.upper()}") == 3 * mult
    for bad in ("", "  ", "kb", "1 xb", "-1 b", "1.5 kb", "9223372036854775808", "9000000000 tb"):
        with pytest.raises(ValueError):
            parse_memory_size(bad)


def value_schema(fields):
    return KeyValueSchema.of(RowType(tuple([DataField("pk", "BIGINT", False)] + list(fields))), ["pk"])


def test_options_parsing():
    o = FileIndexOptions.from_options({
        "file-index.bloom-filter.columns": "a, b,c,",
        "file-index.bloom-filter.a.items": "100", "file-index.bloom-filter.b.fpp": "0.01",
        "file-index.in-manifest-threshold": "1 kb", "file-index.read.enabled": "true",
        "file-index.bloom-filter.a.items.extra": "1",          # not <type>.<column>.<option>: ignored
        "bucket": "4"})
    assert sorted(o.columns) == ["a", "b", "c"]
    assert o.columns["a"] == {"bloom-filter": {"items": "100"}}
    assert o.columns["b"] == {"bloom-filter": {"fpp": "0.01"}}
    assert o.columns["c"] == {"bloom-filter": {}}
    assert o.in_manifest_threshold == 1024
    assert FileIndexOptions.from_options({}).is_empty() and FileIndexOptions.from_options({}).in_manifest_threshold == 500
    with pytest.raises(ValueError, match="should not have empty column"):
        FileIndexOptions.from_options({"file-index.bloom-filter.columns": "a,,b"})
    with pytest.raises(ValueError, match="Can't find top level column options"):
        FileIndexOptions.from_options({"file-index.bloom-filter.columns": "a", "file-index.bloom-filter.z.items": "9"})


def test_container_matches_the_model():
    rng = random.Random(1)
    for names in (["a"], ["x", "é", "z\u0000", "日本", "\U0001F600"], [f"c{i}" for i in range(7)]):
        bodies = {n: bytes(rng.randrange(256) for _ in range(rng.randrange(0, 40))) for n in names}
        got = serialize_file_index({n: {"bloom-filter": b} for n, b in bodies.items()})
        assert got == R.container([(n, [("bloom-filter", b)]) for n, b in bodies.items()])
        assert R.read_container(got) == [(n, {"bloom-filter": b}) for n, b in bodies.items()]
    for s in ("", "abc", "\u0000", "߿", "ࠀ", "￿", "\U0001F600"):
        assert write_utf(s) == R.java_utf(s)


@pytest.mark.parametrize("n", [1, 2, 13, 40])
def test_column_order_is_the_hashmap_order(n):
    rng = random.Random(n)
    names = [f"col_{rng.randrange(10 ** 6)}_{i}" for i in range(n)]
    schema = value_schema([DataField(c, "BIGINT", True) for c in names])
    w = DataFileIndexWriter(schema, FileIndexOptions.from_options({"file-index.bloom-filter.columns": ",".join(names)}))
    want = R.hashmap_buckets(names)
    got, pos = [], 0
    for bucket in want:
        got.append(set(w.columns[pos:pos + len(bucket)]))
        pos += len(bucket)
    assert pos == len(w.columns) and got == want
    # the file column of each spec is its value field behind _KEY_pk, _SEQUENCE_NUMBER and _VALUE_KIND
    assert [s[0] for s in w.specs] == [3 + 1 + names.index(c) for c in w.columns]


class _Files(LocalFileIO):
    def __init__(self):
        self.written = {}

    def write_bytes(self, path, data):
        self.written[path] = data


def test_embedded_up_to_the_threshold_then_a_side_file():
    schema = value_schema([DataField("a", "BIGINT", True)])
    filt = R.filter_of("BIGINT", [1, 2, None], items=100)
    size = len(R.container([("a", [("bloom-filter", filt)])]))
    for threshold, embedded in ((size, True), (size - 1, False)):
        opts = FileIndexOptions.from_options({"file-index.bloom-filter.columns": "a",
                                              "file-index.bloom-filter.a.items": "100",
                                              "file-index.in-manifest-threshold": f"{threshold} b"})
        w = DataFileIndexWriter(schema, opts)
        assert w.sizes == [len(filt)]
        w.build = lambda *args: {"a": filt}                   # the device's part, taken from the model
        io = _Files()
        res = w.write(io, "/d/f.parquet", 0)
        if embedded:
            assert res.embedded_index == R.container([("a", [("bloom-filter", filt)])]) and res.extra_files == []
            assert io.written == {}
        else:
            assert res.embedded_index is None and res.extra_files == ["/d/f.parquet.index"]
            assert R.read_container(io.written["/d/f.parquet.index"]) == [("a", {"bloom-filter": filt})]


REFUSALS = [
    ({"file-index.bitmap.columns": "a"}, N.UnsupportedOnDevice, "bitmap"),
    ({"file-index.bsi.columns": "a"}, N.UnsupportedOnDevice, "bsi"),
    ({"file-index.range-bitmap.columns": "a"}, N.UnsupportedOnDevice, "range-bitmap"),
    ({"file-index.bloom-filter.columns": "m[k]"}, N.UnsupportedOnDevice, "map values"),
    ({"file-index.bloom-filter.columns": "flag"}, ValueError, "^Does not support type boolean$"),
    ({"file-index.bloom-filter.columns": "dec"}, ValueError, "^Does not support decimal$"),
    ({"file-index.bloom-filter.columns": "nope"}, ValueError, "^nope does not exist in column fields$"),
]


def refusal_schema():
    return value_schema([DataField("a", "BIGINT", True), DataField("m", "BIGINT", True),
                         DataField("flag", "BOOLEAN", True), DataField("dec", "DECIMAL(10,2)", True)])


@pytest.mark.parametrize("options,exc,match", REFUSALS)
def test_refusals_come_before_any_device_work(tmp_path, options, exc, match):
    schema = refusal_schema()
    with pytest.raises(exc, match=match) as e:
        KeyValueDataFileWriter(schema, str(tmp_path / "f.parquet"), 1, file_index=FileIndexOptions.from_options(options))
    if exc is ValueError:
        assert not isinstance(e.value, N.UnsupportedOnDevice)
    rewriter = MergeTreeCompactRewriter(schema, DeduplicateMergeFunction.factory(), str(tmp_path),
                                        options=dict(options, **{"file.format": "parquet"}))
    with pytest.raises(exc, match=match):
        rewriter.rewrite_compaction(1, False, [])
    assert os.listdir(tmp_path) == []
