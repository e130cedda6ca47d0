"""LZ4 on the device: Parquet codec 5 pages (Hadoop block / chunk framing, what parquet-mr writes for Paimon's 'lz4')
and ORC CompressionKind 4 chunks.  Hand-built page shapes (dictionary ids, definition levels, small pages, CRCs, V2
pages stored uncompressed under the codec, dictionary pages, pages above 256 KiB whose blocks hold several chunks)
against the builder's values and, where every block is a single chunk, against pyarrow; malformed framing and blocks
refused with PG_ERR_FORMAT; one section mixing codec 5, zstd, Snappy and uncompressed files within and across runs,
with projection; pyarrow.orc LZ4 files of every type; merge-on-read over LZ4 level-0 files and zstd level-1 files; and
the compaction rewriter under 'file.compression.per.level' = '0:lz4,1:zstd' for Parquet and ORC tables."""
import io
import struct

import numpy as np
import pyarrow as pa
import pyarrow.orc as orc
import pyarrow.parquet as pq
import pytest

import parquet_pages as P
from lz4_parquet import HADOOP_LZ4_CHUNK, LZ4, lz4_hadoop, read_struct, to_hadoop_lz4
from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.compact_rewriter import MergeTreeCompactRewriter
from paimon_b200.format import FileFormat, FormatReaderContext, LocalFileIO, read_section
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition, MergeFileSplitRead, concat_batches
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import to_arrow, write_kv_parquet
from test_gpu_orc import all_types_schema, random_batch, write_kv_orc

pytestmark = pytest.mark.gpu

PG_ERR_FORMAT = 6


def _schema(vtype):
    return KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("v", vtype, True))), ["pk"])


def _read_runs(schema, files, n_runs, **kw):
    readers, info = read_section(schema, files, n_runs, **kw)
    out = []
    for r in readers:
        try:
            out.append(r.read_batch())
        finally:
            r.close()
    return out, info


def _single_chunk_blocks(blob: bytes) -> bool:
    """Every Hadoop block of every codec 5 page is one chunk (what Arrow's Hadoop-LZ4 reader takes)."""
    (flen,) = struct.unpack("<I", blob[-8:-4])
    meta, _ = read_struct(blob, len(blob) - 8 - flen)
    for rg in meta[4][1][1]:
        for cc in rg[1][1][1]:
            md = cc[3][1]
            pos = min(md[f][1] for f in (9, 11) if f in md)
            end = pos + md[7][1]
            while pos < end:
                hdr, body0 = read_struct(blob, pos)
                if hdr[2][1] > HADOOP_LZ4_CHUNK:          # (lz4_hadoop cuts chunks of HADOOP_LZ4_CHUNK bytes)
                    return False
                pos = body0 + hdr[3][1]
    return True


# ------------------------------------------------------------------ hand-built codec 5 files

def _lz4_case(case):
    """The builder's uncompressed files with every page recompressed as codec 5."""
    return [to_hadoop_lz4(f) for f in case.files]


LZ4_CASES = {
    "dict_BIGINT": lambda: P.dictionary_case("BIGINT"),        # pages of 74,536 ids and 600 KiB dictionary pages
    "dict_STRING": lambda: P.dictionary_case("STRING"),
    "dict_DOUBLE": lambda: P.dictionary_case("DOUBLE"),
    "rle_boolean": P.rle_boolean_case,
    "def_levels": P.definition_levels_case,
    "small_pages": P.small_pages_case,
    "small_pages_run": P.small_pages_run_case,
    "delta_BIGINT": lambda: P.delta_case("BIGINT"),
}


@pytest.mark.parametrize("name", sorted(LZ4_CASES) + ["headers_lz4"])
def test_codec5_pages_match_the_builder(name):
    if name == "headers_lz4":
        case = P.headers_case(P.UNCOMPRESSED)              # CRCs, statistics, unknown fields, an index page
        files = [to_hadoop_lz4(f, raw_first_v2=True) for f in case.files]
    else:
        case = LZ4_CASES[name]()
        files = _lz4_case(case)
    got, info = _read_runs(_schema(case.vtype), [(f, 0) for f in files], 1)
    vals = P.column_values(got[0].value_column(1), case.vtype)
    assert vals == case.expected, P.first_mismatch(vals, case.expected)
    assert got[0].value_column(0).data[:got[0].n_rows].tolist() == list(range(len(case.expected)))
    assert info.n_data_pages == case.data_pages
    assert info.n_dictionary_pages == (case.dict_pages or 0)
    if all(_single_chunk_blocks(f) for f in files):
        t = pa.concat_tables([pq.read_table(io.BytesIO(f), page_checksum_verification=case.crc) for f in files])
        assert vals == P.arrow_values(t.column("v"), case.vtype)


def test_pages_above_256_kib_hold_several_chunks():
    files = _lz4_case(LZ4_CASES["dict_BIGINT"]())
    assert not _single_chunk_blocks(files[0])


# ------------------------------------------------------------------ malformed codec 5 pages

def _page(stored: bytes, values: bytes, n: int, unc=None) -> P.Page:
    def sub(w):
        w.i32(1, n)
        w.i32(2, P.E_PLAIN)
        w.i32(3, P.E_RLE)
        w.i32(4, P.E_RLE)
    unc = len(values) if unc is None else unc
    return P.Page(P._header(P.DATA_PAGE, unc, len(stored), stored, False, False, 5, sub) + stored, P.DATA_PAGE,
                  P.E_PLAIN, n, unc, len(stored))


def _malformed():
    n = 3000
    values = P.plain(P.INT64, [i * 7 % 1000 for i in range(n)])
    good = lz4_hadoop(values)
    blk = good[8:]
    (ulen,) = struct.unpack(">I", good[:4])
    frames = {
        "truncated": good[:-1],
        "block_length_plus_one": struct.pack(">I", ulen + 1) + good[4:],
        "block_length_minus_one": struct.pack(">I", ulen - 1) + good[4:],
        "chunk_length_past_page": good[:4] + struct.pack(">I", len(blk) + 5) + blk,
        "trailing_bytes": good + b"\x00\x00",
        "offset_zero": None,
        "header_overstates_size": good,
    }
    out = {}
    for name, stored in frames.items():
        unc = None
        if name == "offset_zero":                        # 16 literals, 8 bytes at offset 0, the rest as literals
            rest = len(values) - 24 - 15
            lz = bytes([0xF4, 1]) + values[:16] + b"\x00\x00" + bytes([0xF0]) + b"\xff" * (rest // 255) + \
                bytes([rest % 255]) + values[24:]
            stored = struct.pack(">II", len(values), len(lz)) + lz
        if name == "header_overstates_size":
            unc = len(values) + 8
        page = _page(stored, values, n, unc)
        out[name] = P.kv_file([n], [P.ValueColumn("v", P.INT64, False, [[page]], codec=LZ4)])
    return out


@pytest.mark.parametrize("name", sorted(_malformed()))
def test_malformed_codec5_page_is_a_format_error(name):
    blob = _malformed()[name]
    with pytest.raises(N.PaimonGpuError) as ei:
        _read_runs(_schema("BIGINT"), [(blob, 0)], 1)
    assert ei.value.status == PG_ERR_FORMAT
    case = P.small_pages_case()                           # a good section on the same device still matches
    got, _ = _read_runs(_schema("BIGINT"), [(f, 0) for f in _lz4_case(case)], 1)
    assert P.column_values(got[0].value_column(1), "BIGINT") == case.expected


# ------------------------------------------------------------------ sections mixing codecs

def _write_parquet(run, path, codec, **opts):
    if codec == "lz4":
        write_kv_parquet(run, path, compression="none", **opts)
        blob = to_hadoop_lz4(open(path, "rb").read())
        open(path, "wb").write(blob)
    else:
        write_kv_parquet(run, path, compression=codec, **opts)
    return open(path, "rb").read()


def test_section_mixes_codecs_within_and_across_runs(tmp_path):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    codecs = ["lz4", "zstd", "snappy", "none", "lz4", "lz4", "snappy"]
    runs_of = [0, 0, 0, 1, 1, 2, 2]
    files, plain, parts = [], [], {}
    for i, (codec, r) in enumerate(zip(codecs, runs_of)):
        keys = np.arange(r * 1_000_000 + i * 20_000, r * 1_000_000 + i * 20_000 + 3000 + 1000 * i, dtype=np.int64)
        part = datagen.make_run(schema, r, keys, seed=11, null_prob=0.3, delete_prob=0.1)
        opts = dict(data_page_version="2.0") if i % 2 else dict(use_dictionary=False, data_page_size=4096)
        files.append((_write_parquet(part, str(tmp_path / f"f{i}.parquet"), codec, **opts), r))
        plain.append((_write_parquet(part, str(tmp_path / f"p{i}.parquet"), "none", **opts), r))
        parts.setdefault(r, []).append(part)
    got, info = _read_runs(schema, files, 3)
    assert info.n_files == len(files)
    for r, g in enumerate(got):
        want = concat_batches(schema, parts[r])
        assert g.equals(want), f"run {r}: " + g.first_difference(want)
    mask = [i % 2 == 0 for i in range(schema.n_val)]
    got_p, _ = _read_runs(schema, files, 3, read_value_fields=mask)
    want_p, _ = _read_runs(schema, plain, 3, read_value_fields=mask)
    for r, (g, w) in enumerate(zip(got_p, want_p)):
        assert g.equals(w), f"projected run {r}: " + g.first_difference(w)


# ------------------------------------------------------------------ ORC LZ4

@pytest.mark.parametrize("opts", [dict(compression="lz4"),
                                  dict(compression="lz4", compression_block_size=256 * 1024, stripe_size=64 * 1024),
                                  dict(compression="lz4", dictionary_key_size_threshold=1.0)])
def test_orc_lz4_all_types_against_pyarrow(tmp_path, opts):
    schema = all_types_schema()
    for n, null_p in ((1, 0.0), (33, 0.3), (5000, 0.25), (30000, 0.0), (12000, 0.9)):
        batch = random_batch(schema, n, seed=n + 3, null_p=null_p)
        path = str(tmp_path / f"a{n}.orc")
        write_kv_orc(batch, path, **opts)
        rd = FileFormat.from_identifier("orc").create_reader_factory(schema).create_reader(FormatReaderContext(LocalFileIO(), path))
        try:
            got = rd.read_batch()
        finally:
            rd.close()
        assert got.equals(batch), got.first_difference(batch)


# ------------------------------------------------------------------ merge-on-read and compaction over LZ4 level 0

def _l0_l1_files(tmp_path, schema, fmt):
    rng = np.random.default_rng(17)
    metas, runs = [], []
    l1 = []
    for j in range(3):                                     # level 1: one run of key-disjoint zstd files
        keys = np.arange(j * 4000, j * 4000 + 3500, 2, dtype=np.int64)
        l1.append(datagen.make_run(schema, 0, keys, seed=6, null_prob=0.3))
    for f in range(3):                                     # level 0: overlapping LZ4 files, newer
        keys = np.sort(rng.choice(12000, size=2500, replace=False)).astype(np.int64)
        runs.append(datagen.make_run(schema, f + 1, keys, seed=6, null_prob=0.3, delete_prob=0.15))
    for i, (run, level) in enumerate([(r, 1) for r in l1] + [(r, 0) for r in runs]):
        path = str(tmp_path / f"in-{i}.{fmt}")
        codec = "lz4" if level == 0 else "zstd"
        if fmt == "orc":
            orc.write_table(to_arrow(run), path, compression=codec, stripe_size=64 * 1024)
        else:
            _write_parquet(run, path, codec)
        k = run.columns[0].data
        metas.append(DataFileMeta(path, 0, run.n_rows, int(k[0]), int(k[-1]), level=level))
    return metas, l1 + runs


def _read_all(schema, factory, metas, **kw):
    rd = MergeFileSplitRead(schema, factory).create_merge_reader(metas, **kw)
    batches = []
    while True:
        b = rd.read_batch()
        if b is None:
            break
        batches.append(b)
    rd.close()
    return concat_batches(schema, batches)


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_merge_on_read_over_lz4_level0_and_zstd_level1(tmp_path, fmt):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    metas, file_runs = _l0_l1_files(tmp_path, schema, fmt)
    factory = DeduplicateMergeFunction.factory()
    got = _read_all(schema, factory, metas)
    want = pyoracle.merge(schema, factory.create().with_drop_delete(True), file_runs)
    assert got.equals(want), got.first_difference(want)


@pytest.mark.parametrize("fmt", ["parquet", "orc"])
def test_compaction_reads_lz4_level0_and_writes_zstd(tmp_path, fmt):
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    metas, file_runs = _l0_l1_files(tmp_path, schema, fmt)
    factory = DeduplicateMergeFunction.factory()
    out = tmp_path / "out"
    out.mkdir()
    options = {"file.compression.per.level": "0:lz4,1:zstd", "file.format": fmt}
    rewriter = MergeTreeCompactRewriter(schema, factory, str(out), target_file_rows=1500, options=options)
    result = rewriter.rewrite_compaction(1, False, IntervalPartition(metas).partition())
    assert result.after and all(m.file_name.endswith("." + fmt) for m in result.after)
    for m in result.after:
        if fmt == "parquet":
            md = pq.ParquetFile(m.file_name).metadata
            assert {md.row_group(g).column(c).compression for g in range(md.num_row_groups)
                    for c in range(md.num_columns)} == {"ZSTD"}
        else:
            assert orc.ORCFile(m.file_name).compression == "ZSTD"
    want = pyoracle.merge(schema, factory.create(), file_runs)
    got = _read_all(schema, factory, result.after, keep_delete=True)
    assert got.equals(want), got.first_difference(want)
