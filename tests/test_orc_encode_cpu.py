"""ORC encode, host build: the stream encoders (orc_encode_device.cuh) and the tail writer (orc_meta.cc) that the device
encoder compiles write whole files on the host (tests/native/orc_encode_host_check.cc).  pyarrow.orc and the host build
of the project's ORC decoder both read them back equal to the input; the footers' statistics, read by the wire reader
of orc_stats_reference, match its model.  Also: the table options that choose the format and the ORC codec of a level."""
import ctypes as C
import decimal
import os
import random
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.orc as orc
import pytest

import orc_stats_reference as ref
import orc_util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("orc_enc"))
    so = os.path.join(d, "liborc_enc_host.so")
    csrc = os.path.join(ROOT, "paimon_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + csrc, "-o", so,
                           os.path.join(ROOT, "tests", "native", "orc_encode_host_check.cc"),
                           os.path.join(csrc, "orc_meta.cc")])
    enc = C.CDLL(so)
    enc.orc_enc_host_write.restype = C.c_longlong
    enc.orc_enc_host_write.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_longlong, C.c_longlong, C.c_int, C.c_longlong]
    enc.orc_enc_host_bytes.restype = C.POINTER(C.c_uint8)
    enc.orc_enc_host_error.restype = C.c_char_p
    enc.orc_enc_host_rle2.restype = C.c_int
    enc.orc_enc_host_rle2.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return enc, orc_util.build(d)


# (name, ORC kind, precision, scale, max_length, numpy dtype or None for var-len)
ALL_TYPES = [("k", 4, 0, 0, 0, np.int64), ("t", 1, 0, 0, 0, np.int8), ("s", 2, 0, 0, 0, np.int16),
             ("i", 3, 0, 0, 0, np.int32), ("l", 4, 0, 0, 0, np.int64), ("f", 5, 0, 0, 0, np.float32),
             ("d", 6, 0, 0, 0, np.float64), ("b", 0, 0, 0, 0, np.uint8), ("dt", 15, 0, 0, 0, np.int32),
             ("dec", 14, 15, 4, 0, np.int64), ("str", 7, 0, 0, 0, None), ("vc", 16, 0, 0, 12, None),
             ("bin", 8, 0, 0, 0, None)]


def make_columns(n, null_p, seed):
    rng = np.random.default_rng(seed)
    r = random.Random(seed)
    cols = []
    for name, kind, prec, scale, maxlen, dt in ALL_TYPES:
        valid = np.ones(n, bool) if name == "k" else rng.random(n) >= null_p
        if dt is None:
            if kind == 16:
                vals = ["".join(r.choice("aé€z") for _ in range(r.randrange(0, 13))).encode() for _ in range(n)]
            elif kind == 7:
                vals = [r.choice([b"", b"alpha", b"paimon", b"x" * 40, "üñí".encode()]) for _ in range(n)]
            else:
                vals = [bytes(r.randrange(256) for _ in range(r.randrange(0, 20))) for _ in range(n)]
        elif name == "k":
            vals = np.arange(n, dtype=np.int64) * 3 + 5                     # sorted keys: DELTA runs
        elif dt in (np.float32, np.float64):
            vals = (rng.standard_normal(n) * 1e3).astype(dt)
            if n > 3:
                vals[1], vals[2] = 0.0, -0.0
        elif kind == 0:
            vals = (rng.random(n) < 0.5).astype(np.uint8)
        elif kind == 14:
            vals = rng.integers(-10 ** 14, 10 ** 14, n, dtype=np.int64)
        elif kind == 15:
            vals = rng.integers(-10000, 30000, n).astype(np.int32)
        else:
            info = np.iinfo(dt)
            vals = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
            if n > 40:
                vals[10:20] = 7                                            # SHORT_REPEAT / DELTA runs
        cols.append((name, kind, prec, scale, maxlen, dt, vals, valid))
    return cols


def write(enc, cols, n, stripe_rows, codec=0, block=256 << 10):
    keep = []
    types = np.array([[c[1], c[2], c[3], c[4]] for c in cols], np.int32)
    widths = np.array([0 if c[5] is None else np.dtype(c[5]).itemsize for c in cols], np.int32)
    data = (C.c_void_p * len(cols))()
    offs = (C.c_void_p * len(cols))()
    valid = (C.c_void_p * len(cols))()
    names = (C.c_char_p * len(cols))(*[c[0].encode() for c in cols])
    for i, c in enumerate(cols):
        vals = c[6]
        if c[5] is None:
            o = np.zeros(n + 1, np.int32)
            o[1:] = np.cumsum([len(v) if ok else 0 for v, ok in zip(vals, c[7])]) if n else []
            payload = np.frombuffer(b"".join(v for v, ok in zip(vals, c[7]) if ok) + b"\0", np.uint8)
            keep += [o, payload]
            data[i], offs[i] = payload.ctypes.data, o.ctypes.data
        else:
            a = np.ascontiguousarray(vals)
            keep.append(a)
            data[i] = a.ctypes.data
        v = np.ascontiguousarray(c[7], np.uint8)
        keep.append(v)
        valid[i] = v.ctypes.data
    size = enc.orc_enc_host_write(len(cols), types.ctypes.data, widths.ctypes.data, data, offs, valid, names, n,
                                  stripe_rows, codec, block)
    assert size >= 0, enc.orc_enc_host_error().decode()
    return bytes(enc.orc_enc_host_bytes()[:size])


def want_py(c, i):
    name, kind, prec, scale, maxlen, dt, vals, valid = c
    if not valid[i]:
        return None
    v = vals[i]
    if kind in (7, 16):
        return v.decode()
    if kind == 8:
        return v
    if kind == 0:
        return bool(v)
    if kind == 14:
        return decimal.Decimal(int(v)).scaleb(-scale)
    if kind in (5, 6):
        return float(v)
    return int(v)


def check_round_trip(libs, cols, n, blob, tmp_path):
    enc, dec = libs
    path = str(tmp_path / "t.orc")
    with open(path, "wb") as f:
        f.write(blob)
    table = orc.ORCFile(path).read()
    assert table.num_rows == n and table.column_names == [c[0] for c in cols]
    for c in cols:
        got = table.column(c[0]).to_pylist()
        if c[1] == 15:
            got = table.column(c[0]).cast(pa.int32()).to_pylist()
        want = [want_py(c, i) for i in range(n)]
        if c[1] in (5, 6):
            assert np.array_equal(np.array([np.nan if x is None else x for x in got], c[5]).view(np.uint8),
                                  np.array([np.nan if x is None else x for x in want], c[5]).view(np.uint8)), c[0]
        else:
            assert got == want, c[0]
    widths = [8 if c[1] == 14 else (0 if c[5] is None else np.dtype(c[5]).itemsize) for c in cols]
    rows, got = orc_util.decode(dec, blob, widths)
    assert rows == n
    for c, g in zip(cols, got):
        assert np.array_equal(g[-1], np.asarray(c[7], bool)), c[0]
        if c[5] is None:
            data, offs, _ = g
            assert [bytes(data[offs[i]:offs[i + 1]]) for i in range(n) if c[7][i]] == \
                [v for v, ok in zip(c[6], c[7]) if ok], c[0]
        else:
            vals = g[0].view(c[5]) if c[1] != 0 else g[0]
            assert np.array_equal(vals[c[7]].view(np.uint8), np.asarray(c[6])[c[7]].view(np.uint8)), c[0]


@pytest.mark.parametrize("null_p", [0.0, 0.3, 0.9, 1.0])
@pytest.mark.parametrize("n,stripe_rows", [(0, 64), (1, 64), (37, 8), (1000, 1 << 20), (5000, 1000)])
@pytest.mark.parametrize("codec,block", [(0, 256 << 10), (5, 256 << 10), (5, 1000)])
def test_host_written_files_read_back(libs, tmp_path, null_p, n, stripe_rows, codec, block):
    cols = make_columns(n, null_p, seed=n + int(null_p * 10))
    blob = write(libs[0], cols, n, stripe_rows, codec, block)
    check_round_trip(libs, cols, n, blob, tmp_path)
    if codec == 0:
        _, footer, stripes, whole = ref.read_tail(blob)
        model = [(c[1], c[6], c[7], c[3]) for c in cols]
        want_stripes, want_file = ref.expected(model, n, stripe_rows)
        assert len(stripes) == len(want_stripes)
        for g, (got_s, want_s) in enumerate(zip(stripes, want_stripes)):
            for c, (a, b) in enumerate(zip(got_s, want_s)):
                assert ref.same(a, b), (g, c, a, b)
        for c, (a, b) in enumerate(zip(whole, want_file)):
            assert ref.same(a, b), (c, a, b)


def test_zstd_block_size_splits_streams_and_stores_incompressible_chunks(libs, tmp_path):
    """Random bytes do not compress: their chunks are stored original; repeated bytes are stored compressed."""
    n = 3000
    r = random.Random(3)
    cols = [("k", 4, 0, 0, 0, np.int64, np.arange(n, dtype=np.int64), np.ones(n, bool)),
            ("rnd", 8, 0, 0, 0, None, [bytes(r.randrange(256) for _ in range(50)) for _ in range(n)], np.ones(n, bool)),
            ("rep", 7, 0, 0, 0, None, [b"paimon-orc" * 5] * n, np.ones(n, bool))]
    blob = write(libs[0], cols, n, 1 << 20, codec=5, block=4096)
    check_round_trip(libs, cols, n, blob, tmp_path)
    # walk the chunk headers of the DATA streams: at least one original chunk and one compressed chunk
    orig = comp = 0
    pos = 3
    ps_len = blob[-1]
    end = len(blob) - 1 - ps_len
    while pos < end:
        h = blob[pos] | blob[pos + 1] << 8 | blob[pos + 2] << 16
        length = h >> 1
        if length > 4096 or pos + 3 + length > end:
            break
        orig += h & 1
        comp += not h & 1
        pos += 3 + length
    assert orig > 0 and comp > 0


def rle2(enc, values, signed=1):
    v = np.ascontiguousarray(values, np.int64)
    dst = np.zeros(16 + 9 * len(v), np.uint8)
    form, width = C.c_int(0), C.c_int(0)
    size = enc.orc_enc_host_rle2(v.ctypes.data, len(v), signed, dst.ctypes.data, C.byref(form), C.byref(width))
    return form.value, width.value, size


def test_rle2_run_forms(libs):
    enc = libs[0]
    assert rle2(enc, [5] * 3)[0] == 0 and rle2(enc, [5] * 10)[0] == 0            # SHORT_REPEAT at lengths 3 and 10
    assert rle2(enc, [5] * 11)[0] == 3                                             # fixed DELTA beyond 10
    assert rle2(enc, [5] * 2)[0] == 1                                              # too short for either
    assert rle2(enc, np.arange(100) * -7)[:2] == (3, 0)                            # fixed negative delta
    assert rle2(enc, -np.cumsum(np.arange(100) % 5))[0] == 3                       # variable negative deltas
    i64 = np.iinfo(np.int64)
    assert rle2(enc, [i64.min, i64.max, i64.min])[0] == 1                          # deltas overflow int64: DIRECT
    assert rle2(enc, [0, i64.max, i64.max])[0] in (1, 3)
    for w in range(1, 64):                                                         # DIRECT at every width
        rng = np.random.default_rng(w)
        v = rng.integers(0, 1 << w, 300, dtype=np.uint64, endpoint=False).astype(np.int64) if w < 63 else \
            rng.integers(i64.min, i64.max, 300)
        form, width, _ = rle2(enc, v, 0 if w < 63 else 1)
        assert form in (1, 3)


def test_integer_and_byte_edges_round_trip(libs, tmp_path):
    i64 = np.iinfo(np.int64)
    n = 4096
    rng = np.random.default_rng(9)
    widths = [rng.integers(0, 1 << w, 64).astype(np.int64) - (1 << (w - 1)) for w in range(1, 63)]
    edge = np.concatenate([[i64.min, i64.max, i64.min, 0, i64.max] * 3, [7] * 3, [8] * 10, [9] * 11,
                           np.arange(600) * -3, np.cumsum(rng.integers(0, 1 << 40, 600)), *widths])
    edge = np.resize(edge, n).astype(np.int64)
    kinds = np.resize(np.repeat(np.array([0, 0, 0, 1, 2, 3], np.int8), [127, 128, 129, 3, 5, 200]), n)
    cols = [("l", 4, 0, 0, 0, np.int64, edge, np.ones(n, bool)),
            ("kind", 1, 0, 0, 0, np.int8, kinds, np.ones(n, bool)),
            ("lnull", 4, 0, 0, 0, np.int64, edge[::-1].copy(), rng.random(n) > 0.5)]
    for codec in (0, 5):
        blob = write(libs[0], cols, n, 1024, codec)
        check_round_trip(libs, cols, n, blob, tmp_path)


# ---- table options


def test_format_for_level():
    from paimon_b200.compact_rewriter import format_for_level
    assert format_for_level(None, 3) == "parquet"
    assert format_for_level({"file.format": "ORC"}, 3) == "orc"
    opts = {"file.format": "orc", "file.format.per.level": "0:avro,5:parquet"}
    assert [format_for_level(opts, lv) for lv in (0, 1, 5)] == ["avro", "orc", "parquet"]
    assert format_for_level({"file.format.per.level": {0: "orc"}}, 0) == "orc"


def test_orc_compression_for_level():
    from paimon_b200.compact_rewriter import orc_compression_for_level
    assert orc_compression_for_level(None, 0) == ("zstd", 1, 0)
    assert orc_compression_for_level({"file.compression": "none"}, 0) == ("none", 1, 0)
    opts = {"file.compression": "zstd", "file.compression.per.level": "0:lz4", "file.compression.zstd-level": "-3"}
    assert orc_compression_for_level(opts, 0) == ("lz4", -3, 0)
    assert orc_compression_for_level(opts, 2) == ("zstd", -3, 0)
    opts.update({"orc.compress": "NONE", "orc.compression.zstd.level": "1", "orc.compress.size": "65536"})
    assert orc_compression_for_level(opts, 0) == ("none", 1, 65536)


def test_orc_column_types():
    from paimon_b200.types import orc_column_type
    assert orc_column_type("DECIMAL(12,3)") == (14, 12, 3, 0)
    assert orc_column_type("VARCHAR(24)") == (16, 0, 0, 24)
    assert orc_column_type("VARCHAR(2147483647)") == (7, 0, 0, 0)
    assert [orc_column_type(t)[0] for t in ("TINYINT", "SMALLINT", "INT", "TIME", "BIGINT", "FLOAT", "DOUBLE",
                                            "BOOLEAN", "DATE", "STRING", "BINARY(4)", "VARBINARY(9)")] == \
        [1, 2, 3, 3, 4, 5, 6, 0, 15, 7, 8, 8]
