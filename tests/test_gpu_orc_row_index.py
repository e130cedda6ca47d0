"""ORC row indexes and bloom filters written on the device (pg_orc_encode_indexed), against the model in
tests/orc_index_reference.py: every file reads back equal to the batch through pyarrow.orc and pg_orc_read_section;
every entry's statistics equal the model's; every position, decoded from where it points (byte RLE, boolean bits, RLE v2
SHORT_REPEAT / DIRECT / DELTA, raw values; ZSTD chunks inflated by the host zstd decoder), gives the row group's first
values; every BLOOM_FILTER_UTF8 filter equals the model's bits.  Also: a NULL index and a stride of 0 give
pg_orc_encode's bytes, the refusals, and MergeTreeCompactRewriter(row_index=True)."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import codec_filter
import orc_index_reference as X
import orc_stats_reference as ref
from codec_corpora import ZSTD
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.compact_rewriter import MergeTreeCompactRewriter, file_column_names
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import IntervalPartition
from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle
from paimon_b200.types import orc_column_type
from test_gpu_orc_write import _files, all_types_schema, check_file, encode, model_columns, random_rows, slice_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def codec(tmp_path_factory):
    return codec_filter.build(str(tmp_path_factory.mktemp("zs")))


def frames_of(blob, codec):
    """frame bytes -> inflated bytes for every compressed chunk of a ZSTD file (the body is chunks back to back)"""
    end = len(blob) - 1 - blob[-1]
    pos, frames = 3, []
    while pos < end:
        h = blob[pos] | blob[pos + 1] << 8 | blob[pos + 2] << 16
        if not h & 1:
            frames.append(bytes(blob[pos + 3:pos + 3 + (h >> 1)]))
        pos += 3 + (h >> 1)
    out = codec([(ZSTD, f, 1 << 23) for f in frames])
    assert all(r >= 0 for r, _ in out)
    return {f: o for f, (_, o) in zip(frames, out)}


# ---- decoders of the first values at a position


def byte_rle(b, n):
    out, p = [], 0
    while len(out) < n:
        h = b[p]
        if h < 128:
            out += [b[p + 1]] * (h + 3)
            p += 2
        else:
            out += list(b[p + 1:p + 1 + 256 - h])
            p += 1 + 256 - h
    return out[:n]


_W = list(range(1, 25)) + [26, 28, 30, 32, 40, 48, 56, 64]


def _uvarint(b, p):
    v, sh = 0, 0
    while True:
        x = b[p]
        p += 1
        v |= (x & 0x7F) << sh
        sh += 7
        if not x & 0x80:
            return v, p


def _unzz(v):
    return (v >> 1) ^ -(v & 1)


def _bits(b, p, n, w):
    acc = int.from_bytes(b[p:p + (n * w + 7) // 8], "big")
    total = ((n * w + 7) // 8) * 8
    return [(acc >> (total - (i + 1) * w)) & ((1 << w) - 1) for i in range(n)], p + (n * w + 7) // 8


def rle2(b, n, signed):
    out, p = [], 0
    while len(out) < n:
        h = b[p]
        enc = h >> 6
        if enc == 0:                                          # SHORT_REPEAT
            w, cnt = ((h >> 3) & 7) + 1, (h & 7) + 3
            v = int.from_bytes(b[p + 1:p + 1 + w], "big")
            out += [_unzz(v) if signed else v] * cnt
            p += 1 + w
        elif enc == 1:                                        # DIRECT
            w, cnt = _W[(h >> 1) & 31], ((h & 1) << 8 | b[p + 1]) + 1
            vals, p = _bits(b, p + 2, cnt, w)
            out += [_unzz(v) if signed else v for v in vals]
        elif enc == 3:                                        # DELTA
            code, cnt = (h >> 1) & 31, ((h & 1) << 8 | b[p + 1]) + 1
            base, p = _uvarint(b, p + 2)
            base = _unzz(base) if signed else base
            db, p = _uvarint(b, p)
            db = _unzz(db)
            vals = [base, base + db]
            if code == 0:
                vals = [base + i * db for i in range(cnt)]
            else:
                deltas, p = _bits(b, p, cnt - 2, _W[code])
                for d in deltas:
                    vals.append(vals[-1] + (d if db >= 0 else -d))
            out += vals[:cnt]
        else:
            raise AssertionError("PATCHED_BASE is not written")
    return out[:n]


def stream_at(st, col, skind, pos, i, zstd, frames):
    stored = st.streams[(col + 1, skind)]
    if zstd:
        raw = X.inflate(stored[pos[i]:], 5, frames.__getitem__)
        return raw[pos[i + 1]:], i + 2
    return stored[pos[i]:], i + 1


def check_group(st, g, col, kind, vals, valid, scale, g0, r0, r1, zstd, frames):
    pos = st.index[col + 1][g][0]
    i = 0
    if (col + 1, X.PRESENT) in st.streams:
        b, i = stream_at(st, col, X.PRESENT, pos, i, zstd, frames)
        assert pos[i:i + 2] == [0, 0]
        i += 2
        m = min(8, r1 - r0)
        first = byte_rle(b, 1)[0]
        assert [bool(first >> (7 - j) & 1) for j in range(m)] == list(valid[r0:r0 + m]), (col, g)
    rows = [r for r in range(r0, r1) if valid[r]][:4]
    m = len(rows)
    b, i = stream_at(st, col, X.DATA, pos, i, zstd, frames)
    if kind == 0:                                             # BOOLEAN: [offset, 0, bit]
        assert pos[i] == 0
        bit = pos[i + 1]
        i += 2
        assert bit == int(valid[g0:r0].sum()) % 8
        by = byte_rle(b, (bit + m + 7) // 8)
        got = [bool(by[(bit + j) >> 3] >> (7 - ((bit + j) & 7)) & 1) for j in range(m)]
        assert got == [bool(vals[r]) for r in rows], (col, g)
    elif kind == 1:
        assert pos[i] == 0
        i += 1
        assert [x if x < 128 else x - 256 for x in byte_rle(b, m)] == [int(vals[r]) for r in rows], (col, g)
    elif kind in (2, 3, 4, 15):
        assert pos[i] == 0
        i += 1
        assert rle2(b, m, True) == [int(vals[r]) for r in rows], (col, g)
    elif kind in (5, 6):
        w = 4 if kind == 5 else 8
        got = [b[w * j:w * j + w] for j in range(m)]
        assert got == [np.asarray(vals[r]).tobytes() for r in rows], (col, g)
    elif kind in X.BYTES_KINDS:
        if m:
            assert b[:len(vals[rows[0]])] == vals[rows[0]], (col, g)
        lb, i = stream_at(st, col, X.LENGTH, pos, i, zstd, frames)
        assert pos[i] == 0
        i += 1
        assert rle2(lb, m, False) == [len(vals[r]) for r in rows], (col, g)
    elif kind == X.DECIMAL:
        p, got = 0, []
        for _ in range(m):
            v, p = _uvarint(b, p)
            got.append(_unzz(v))
        assert got == [int(vals[r]) for r in rows], (col, g)
        sb, i = stream_at(st, col, X.SECONDARY, pos, i, zstd, frames)
        assert pos[i] == 0
        i += 1
        assert rle2(sb, m, True) == [scale] * m, (col, g)
    assert i == len(pos), (col, g, pos)


def check_index(schema, batch, path, stripe_rows, stride, bloom_cols, fpp, zstd, codec):
    blob = open(path, "rb").read()
    frames = frames_of(blob, codec) if zstd else {}
    got_stride, stripes = X.read_file(blob, frames.__getitem__)
    assert got_stride == stride
    n = batch.n_rows
    model = model_columns(schema, batch)
    groups = X.row_groups(n, stripe_rows, stride)
    want = X.expected_entries(model, n, stripe_rows, stride)
    assert len(stripes) == len(groups)
    bits, k = X.sizing(stride, fpp) if bloom_cols else (0, 0)
    for st, gr, w in zip(stripes, groups, want):
        ncol = len(model) + 1                                   # the index streams first: root, then per column
        want_order = [(kd, c) for c in range(ncol) for kd in ([6, 8] if c - 1 in bloom_cols else [6])]
        assert st.order[:len(want_order)] == want_order
        assert all(kind not in (6, 8) for kind, _ in st.order[len(want_order):])
        for c in range(ncol):
            assert len(st.index[c]) == len(gr)
            for g, ((_, s), ws) in enumerate(zip(st.index[c], w[c])):
                assert ref.same(s, ws), (c, g, s, ws)
        assert all(not p for p, _ in st.index[0])
        g0 = gr[0][0]
        for c, (kind, vals, valid, scale) in enumerate(model):
            for g, (r0, r1) in enumerate(gr):
                check_group(st, g, c, kind, vals, valid, scale, g0, r0, r1, zstd, frames)
            if c in bloom_cols:
                assert [f[0] for f in st.bloom[c + 1]] == [k] * len(gr)
                for g, (r0, r1) in enumerate(gr):
                    assert st.bloom[c + 1][g][1] == X.bloom_bitset(X.hashes(kind, vals[r0:r1], valid[r0:r1]), bits, k)
            else:
                assert c + 1 not in st.bloom


def _bloomable(schema):
    return [i for i, f in enumerate(schema.file_fields()) if orc_column_type(f.type)[0] not in (0, 14)]


@pytest.mark.parametrize("case", [
    dict(n=25300, null_p=0.3, stripe_rows=12000, stride=1000, compression="none", fpp=0.05),
    dict(n=25300, null_p=0.3, stripe_rows=12000, stride=1000, compression="zstd", compression_block_size=2000, fpp=0.05),
    dict(n=60000, null_p=0.0, stripe_rows=25000, stride=10000, compression="zstd", fpp=0.01),
    dict(n=23000, null_p=1.0, stripe_rows=0, stride=10000, compression="none", fpp=0.01),
])
def test_all_types_row_index(tmp_path, codec, case):
    case = dict(case)
    n, null_p, fpp = case.pop("n"), case.pop("null_p"), case.pop("fpp")
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(n), n, null_p))
    names = [f.name for f in schema.value_type.fields if orc_column_type(f.type)[0] not in (0, 14)]
    bloom = [schema.n_key + 2 + i for i, f in enumerate(schema.value_type.fields) if f.name in names]
    path = str(tmp_path / "idx.orc")
    written = encode(schema, batch, path, row_index_stride=case["stride"], bloom_filter_columns=names,
                     bloom_filter_fpp=fpp, stripe_rows=case["stripe_rows"], compression=case["compression"],
                     compression_block_size=case.get("compression_block_size", 0))
    check_file(schema, batch, path, written, case["stripe_rows"])
    check_index(schema, batch, path, case["stripe_rows"] or 1 << 20, case["stride"], bloom, fpp,
                case["compression"] == "zstd", codec)


@pytest.mark.parametrize("compression", ["none", "zstd"])
def test_slice_of_a_run(tmp_path, codec, compression):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    run = datagen.make_runs(schema, 1, 30000, seed=4, null_prob=0.4, delete_prob=0.1)[0]
    path = str(tmp_path / "s.orc")
    bloom_names = [f.name for f in schema.value_type.fields]
    written = encode(schema, run, path, 16, 12000, stripe_rows=8192, compression=compression, row_index_stride=1000,
                     bloom_filter_columns=bloom_names, bloom_filter_fpp=0.05)
    part = slice_batch(schema, run, 16, 12016)                 # of 15000 rows
    check_file(schema, part, path, written, 8192)
    check_index(schema, part, path, 8192, 1000, list(range(schema.n_key + 2, len(schema.file_fields()))), 0.05,
                compression == "zstd", codec)


def _encode_bytes(lib, h, names, opts, index, use_plain=False):
    fh = C.c_uint64(0)
    if use_plain:
        st = lib.pg_orc_encode(h, names, 0, -1, C.byref(opts), C.byref(fh))
    else:
        st = lib.pg_orc_encode_indexed(h, names, 0, -1, C.byref(opts), C.byref(index) if index else None, C.byref(fh))
    if st:
        return st
    meta = N.PgFileMeta()
    N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
    buf = np.empty(meta.file_bytes, np.uint8)
    N.check(lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
    lib.pg_parquet_file_free(fh.value)
    return buf.tobytes()


def test_no_index_bytes_and_refusals():
    schema = all_types_schema()
    batch = KeyValueBatch.from_rows(schema, random_rows(random.Random(2), 5000, 0.2))
    lib = N.init(0)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[x.encode() for x in names])
    fields = schema.file_fields()
    types = (N.PgOrcColumnType * len(fields))(*[N.PgOrcColumnType(*orc_column_type(f.type)) for f in fields])
    col = {f.name: i for i, f in enumerate(fields)}
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    try:
        h = rd._open(sh.handle)
        for comp in (0, 5):
            opts = N.PgOrcWriteOptions(2048, comp, 1, 0, types)
            plain = _encode_bytes(lib, h, arr, opts, None, use_plain=True)
            assert isinstance(plain, bytes)
            assert _encode_bytes(lib, h, arr, opts, None) == plain
            assert _encode_bytes(lib, h, arr, opts, N.PgOrcIndexOptions(0, 0, None, 0.0)) == plain
            indexed = _encode_bytes(lib, h, arr, opts, N.PgOrcIndexOptions(1000, 0, None, 0.0))
            assert isinstance(indexed, bytes) and indexed != plain

        opts = N.PgOrcWriteOptions(0, 0, 1, 0, types)

        def run(stride, cols=(), fpp=0.01, n=None):
            a = (C.c_int32 * max(len(cols), 1))(*cols)
            return _encode_bytes(lib, h, arr, opts, N.PgOrcIndexOptions(stride, len(cols) if n is None else n, a, fpp))
        s = col["str"]
        assert isinstance(run(1000, [s, col["l"], col["d"], col["f"], col["dt"], col["bin"], col["t"]]), bytes)
        for bad in (run(999), run(-8), run(0, [s]), run(1000, [s], 0.0), run(1000, [s], 1.0), run(1000, [s, s]),
                    run(1000, [len(fields)]), run(1000, [-1]), run(1000, [s], n=-1)):
            assert bad == 1
        for bad in (run(1004), run(1000, [col["b"]]), run(1000, [col["dec"]]), run(10 ** 6, [s], 1e-6)):
            assert bad == 2
    finally:
        rd.close()
        sh.close()


def test_compact_rewriter_row_index(tmp_path):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    metas, _ = _files(tmp_path, schema, [(0, 4000), (6000, 9000)], 4, 7)
    factory = DeduplicateMergeFunction.factory()
    options = {"file.format": "parquet", "file.format.per.level": "5:orc", "orc.row.index.stride": "1000",
               "orc.bloom.filter.columns": schema.value_type.fields[1].name, "orc.bloom.filter.fpp": "0.05",
               "file.compression": "none"}
    sections = IntervalPartition(metas).partition()
    out = {}
    for flag in (False, True):
        for level in (5, 1):
            d = tmp_path / f"{flag}-{level}"
            os.makedirs(str(d))
            res = MergeTreeCompactRewriter(schema, factory, str(d), target_file_rows=3000, options=options,
                                           row_index=flag).rewrite_compaction(level, False, sections)
            out[flag, level] = [open(m.file_name, "rb").read() for m in res.after]
    assert out[True, 1] == out[False, 1]                         # Parquet levels ignore row_index
    for plain, indexed in zip(out[False, 5], out[True, 5]):
        assert X.read_file(plain)[0] == 0
        stride, stripes = X.read_file(indexed)
        assert stride == 1000 and all(st.bloom.keys() == {schema.n_key + 4} for st in stripes)   # ORC column ids
        assert all(st.index_length > 0 for st in stripes)
    bad = dict(options, **{"orc.row.index.stride": "1004"})
    with pytest.raises(N.UnsupportedOnDevice):
        MergeTreeCompactRewriter(schema, factory, str(tmp_path), options=bad, row_index=True).rewrite_compaction(
            5, False, sections)
