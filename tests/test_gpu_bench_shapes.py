"""The decode and rewrite paths at bench.py's own shapes, every column checked bit for bit (the inputs are restated in
tests/bench_shapes.py and held to the bench by test_bench_shapes_cpu.py).

  C5   the lineitem bucket pyarrow writes (15.6 M rows, 5 runs, dictionary pages with PLAIN fallback pages behind them,
       800 000-row row groups), `none` and zstd-1: every decoded run against pyarrow's read of the same bytes, the
       deduplicate merge against the oracle's merge of pyarrow's runs.
  C3   `--source parquet`: runs written by the device encoder with 20 000-row pages and 400 000-row row groups, two
       full row groups and a short last one ending in a short page, decoded as one section.
  C4   the rewrite: 32 runs x 500 000 rows, 5 % deletes, drop-delete, merged and encoded as Parquet (the bench's call,
       and zstd) and as ORC (uncompressed and zstd) at the default row-group and stripe sizes; every file read back by
       pyarrow and by the device decoder, its statistics held to the models, and every zstd frame equal to the one the
       host build of the frame encoder writes for the same bytes.  MergeTreeCompactRewriter at the same size.
Needs an H100."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.orc as orc
import pyarrow.parquet as pq
import pytest

import bench_shapes as B
import page_index_reference as P
import stats_reference as S
from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.compact_rewriter import KeyValueDataFileWriter, MergeTreeCompactRewriter, file_column_names
from paimon_b200.format import FileFormat, FileUpload, FormatReaderContext, LocalFileIO, read_section
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.merge_tree_readers import IntervalPartition
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader, _SchemaHandle

from parquet_util import arrow_to_batch
from test_gpu_orc_write import _chunks, _read_all, check_file, read_device
from test_gpu_parquet_write_stats import _raw_of_model, footer_of
from test_gpu_parquet_write_zstd import ZSTD, pages_of
from test_zstd_encode_cpu import compress, zse  # noqa: F401  (zse: the host build of the encoder, a fixture)

pytestmark = pytest.mark.gpu

PLAIN, PLAIN_DICTIONARY, RLE_DICTIONARY = 0, 2, 8
DATA_PAGE, DICTIONARY_PAGE = 0, 2


def names_array(schema):
    names = file_column_names(schema)
    return (C.c_char_p * len(names))(*[n.encode() for n in names])


def read_parquet_bytes(schema, buf):
    return arrow_to_batch(schema, pq.read_table(pa.BufferReader(pa.py_buffer(buf))))


def frame_content_size(frame):
    """Frame_Content_Size of a zstd frame header (RFC 8878 3.1.1.1)."""
    fhd = frame[4]
    single, did, fcs = fhd >> 5 & 1, fhd & 3, fhd >> 6
    pos = 5 + (1 - single) + (0, 1, 2, 4)[did]
    size = (single, 2, 4, 8)[fcs]
    v = int.from_bytes(bytes(frame[pos:pos + size]), "little")
    return v + 256 if size == 2 else v


def assert_host_build_frame(zse, frame, what):
    """The device's frame decompresses (libzstd) to some bytes; the host build's frame of those bytes is the same."""
    body = ZSTD.decompress(frame, decompressed_size=frame_content_size(frame), asbytes=True)
    assert compress(zse, body) == bytes(frame), f"{what}: device and host frames of {len(body)} bytes differ"


def data_page_encodings(buf):
    """{(row group, column): (has a dictionary page, [encoding of every data page])} of a Parquet file, from the
    footer's chunk offsets and every page header."""
    md = pq.ParquetFile(pa.BufferReader(pa.py_buffer(buf))).metadata
    mv = memoryview(buf)
    out = {}
    for g in range(md.num_row_groups):
        for c in range(md.num_columns):
            cc = md.row_group(g).column(c)
            off = cc.dictionary_page_offset if cc.has_dictionary_page else cc.data_page_offset
            end = off + cc.total_compressed_size
            has_dict, encs = False, []
            while off < end:
                h, hend = P.read_struct(mv, off)
                if h[1] == DICTIONARY_PAGE:
                    has_dict = True
                elif h[1] == DATA_PAGE:
                    encs.append(h[5][2])
                off = hend + h[3]
            assert off == end
            out[(g, c)] = (has_dict, encs)
    return md, out


# ---------------------------------------------------------------------------------------------- C5

@pytest.mark.parametrize("codec", ["none", "zstd"])
def test_c5_decode_and_merge_every_column(codec):
    schema = B.schema_c5()
    names = file_column_names(schema)
    files, n_in, _ = B.c5_bucket(schema, codec)
    # the edges are reached: dictionary pages, chunks whose data pages go from dictionary ids to PLAIN after the
    # 1 MiB dictionary limit, several row groups
    md, pages = data_page_encodings(files[0][0])
    assert md.num_row_groups > 1
    assert any(d for d, _ in pages.values())
    for name in ("l_partkey", "l_comment"):
        c = names.index(name)
        mixed = [g for (g, cc), (d, encs) in pages.items() if cc == c and d and PLAIN in encs
                 and ({PLAIN_DICTIONARY, RLE_DICTIONARY} & set(encs))]
        assert mixed, f"{name}: no chunk with dictionary and PLAIN data pages"
    want_runs = [read_parquet_bytes(schema, buf) for buf, _ in files]
    assert sum(r.n_rows for r in want_runs) == n_in
    up = FileUpload(files, 0)
    try:
        readers, info = read_section(schema, up.wait(), len(files))
        assert info.n_rows == n_in and info.n_dictionary_pages > 0
        rd = SortMergeReader(readers, DeduplicateMergeFunction.factory().create(), None, 0)
        try:
            for r, (reader, want) in enumerate(zip(readers, want_runs)):
                got = reader.read_batch()
                assert got.equals(want), f"run {r}: {got.first_difference(want)}"
                del got
            rd.execute()
            merged = rd.fetch()
        finally:
            rd.close()
    finally:
        up.close()
    want = pyoracle.merge(schema, DeduplicateMergeFunction.factory().create(), want_runs, pyoracle.SORT_LOSER_TREE)
    assert merged.n_rows == want.n_rows == want_runs[0].n_rows
    assert merged.equals(want), merged.first_difference(want)


# ---------------------------------------------------------------------------------------------- C3 --source parquet

def test_c3_parquet_source_round_trip():
    """4 C3 runs of 923 457 rows: row groups of 400 000, 400 000 and 123 457 rows, the last one ending in a
    3 457-row page.  Every run decoded from its device image in one section equals its source."""
    schema = datagen.schema_c3()
    page, group = B.PARQUET_PAGE_ROWS, B.PARQUET_GROUP_ROWS
    per_run = 2 * group + 6 * page + 3457
    n_runs = 4
    runs = datagen.make_runs(schema, n_runs, n_runs * per_run, seed=43, null_prob=B.WORKLOADS["c3"]["null_prob"])
    assert all(r.n_rows == per_run for r in runs)
    groups = S.row_groups(per_run, page, group)
    assert [b - a for a, b in groups] == [group, group, 6 * page + 3457]
    n_pages = sum(-(-(b - a) // page) for a, b in groups) * schema.n_cols
    lib = N.init(0)
    arr = names_array(schema)
    sh = _SchemaHandle(schema, 0)
    handles, images = [], []
    try:
        for i, run in enumerate(runs):
            src = SortedRunReader(schema, run)
            try:
                fh = C.c_uint64(0)
                opts = N.PgParquetWriteOptions(group, page)
                N.check(lib.pg_parquet_encode(src._open(sh.handle), arr, 0, -1, C.byref(opts), C.byref(fh)))
                handles.append(fh.value)
            finally:
                src.close()
            meta = N.PgFileMeta()
            N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
            assert (meta.n_rows, meta.n_pages) == (per_run, n_pages)
            ptr, size = C.c_void_p(0), C.c_int64(0)
            N.check(lib.pg_parquet_file_device_image(fh.value, C.byref(ptr), C.byref(size)))
            images.append(((ptr.value, size.value), i))
            if i == 0:                                   # the short last page, from the page headers
                buf = np.zeros(meta.file_bytes, np.uint8)
                N.check(lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
                blob = buf.tobytes()
                del buf
                chunks = P.footer_chunks(blob)
                assert len(chunks) == 3
                for (a, b), row in zip(groups, chunks):
                    off, counts = row[0].data_page_offset, []
                    while off < row[0].data_page_offset + row[0].total_compressed_size:
                        hl, comp, nv = P.page_header(blob, off)
                        counts.append(nv)
                        off += hl + comp
                    assert counts == [min(page, b - x) for x in range(a, b, page)]
        readers, info = read_section(schema, images, n_runs)
        try:
            assert info.n_rows == n_runs * per_run
            for r, (reader, want) in enumerate(zip(readers, runs)):
                got = reader.read_batch()
                assert got.equals(want), f"run {r}: {got.first_difference(want)}"
                del got
        finally:
            for reader in readers:
                reader.close()
    finally:
        for fh in handles:
            lib.pg_parquet_file_free(fh)
        sh.close()


# ---------------------------------------------------------------------------------------------- C4 rewrite

@pytest.fixture(scope="module")
def c4():
    """(schema, drop-delete spec, the 32 runs, the oracle's merge)"""
    schema = B.schema_c4()
    w = B.WORKLOADS["c4"]
    runs = datagen.make_runs(schema, w["n_runs"], w["rows"], seed=44, null_prob=w["null_prob"],
                             delete_prob=w["delete_prob"])
    assert [r.n_rows for r in runs] == [w["rows"] // w["n_runs"]] * w["n_runs"]
    spec = DeduplicateMergeFunction.factory().create().with_drop_delete()
    want = pyoracle.merge(schema, spec, runs, pyoracle.SORT_LOSER_TREE)
    return schema, spec, runs, want


@pytest.fixture(scope="module")
def c4_merge(c4):
    """The merge handle holding the merged batch, as the bench encodes it."""
    schema, spec, runs, _ = c4
    rd = SortMergeReader.create_sort_merge_reader([SortedRunReader(schema, b) for b in runs], None, None, spec)
    try:
        rd.execute()
        yield rd
    finally:
        rd.close()


def test_c4_merge_at_full_size(c4, c4_merge):
    _, _, _, want = c4
    got = c4_merge.fetch()
    assert got.n_rows == want.n_rows
    assert got.equals(want), got.first_difference(want)


def _encode_parquet(schema, h, codec):
    """pg_parquet_encode with NULL options (the bench's call), or pg_parquet_encode_compressed zstd-1 with NULL
    options -> (file bytes, pg_file_meta, [(null_count, has_min_max, min8, max8)] of every column)"""
    lib = N.init(0)
    fh = C.c_uint64(0)
    if codec is None:
        N.check(lib.pg_parquet_encode(h, names_array(schema), 0, -1, None, C.byref(fh)))
    else:
        N.check(lib.pg_parquet_encode_compressed(h, names_array(schema), 0, -1, None, codec, 1, C.byref(fh)))
    try:
        meta = N.PgFileMeta()
        N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
        buf = np.zeros(meta.file_bytes, np.uint8)
        N.check(lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
        cols = []
        for c in range(schema.n_cols):
            nulls, has = C.c_int64(0), C.c_int32(0)
            mn, mx = np.zeros(1, np.int64), np.zeros(1, np.int64)
            N.check(lib.pg_parquet_file_column_stats(fh.value, c, C.byref(nulls), C.byref(has), mn.ctypes.data,
                                                     mx.ctypes.data))
            cols.append((int(nulls.value), bool(has.value), mn.tobytes(), mx.tobytes()))
        return buf.tobytes(), meta, cols
    finally:
        lib.pg_parquet_file_free(fh.value)


@pytest.mark.parametrize("codec", [None, 6], ids=["none", "zstd"])
def test_c4_rewrite_as_parquet(c4, c4_merge, tmp_path, zse, codec):
    schema, _, _, want = c4
    n = want.n_rows
    types = schema.physical_types()
    file_bytes, meta, cols = _encode_parquet(schema, c4_merge._merge_h, codec)
    path = str(tmp_path / "c4.parquet")
    with open(path, "wb") as f:
        f.write(file_bytes)
    # the shape: several row groups at the default size
    groups = S.row_groups(n)
    assert len(groups) >= 2 and pq.ParquetFile(path).metadata.num_row_groups == len(groups)
    # both readers
    got = arrow_to_batch(schema, pq.read_table(path))
    assert got.equals(want), got.first_difference(want)
    del got
    rd = FileFormat.from_identifier("parquet").create_reader_factory(schema).create_reader(
        FormatReaderContext(LocalFileIO(), path))
    try:
        dev = rd.read_batch()
    finally:
        rd.close()
    assert dev.equals(want), dev.first_difference(want)
    del dev
    # pg_file_meta, the footer statistics of every chunk, the file statistics of every column
    m = S.data_file_meta(want)
    assert (meta.n_rows, meta.delete_row_count, meta.min_sequence_number, meta.max_sequence_number) == \
        (m.row_count, m.delete_row_count, m.min_sequence_number, m.max_sequence_number)
    assert footer_of(file_bytes, types) == S.footer_stats(want)
    for c, (t, raw, w) in enumerate(zip(types, cols, S.file_stats(want))):
        model = _raw_of_model(t, w)
        assert raw[:2] == model[:2] and (not raw[1] or raw[2:] == model[2:]), (c, raw, w)
    if codec is not None:
        frames = pages_of(file_bytes)
        assert len(frames) == meta.n_pages
        for p, (_, frame) in enumerate(frames):
            assert_host_build_frame(zse, frame, f"page {p}")


@pytest.mark.parametrize("compression", ["none", "zstd"])
def test_c4_rewrite_as_orc(c4, c4_merge, tmp_path, zse, compression):
    schema, _, _, want = c4
    path = str(tmp_path / "c4.orc")
    written = KeyValueDataFileWriter(schema, path, 5, file_format="orc", compression=compression).write(
        c4_merge._merge_h)
    check_file(schema, want, path, written, 0)
    assert orc.ORCFile(path).nstripes == len(S.row_groups(want.n_rows)) >= 2      # 1 Mi-row stripes
    if compression == "zstd":
        blob = open(path, "rb").read()
        compressed = [(ln, at) for orig, ln, at in _chunks(blob, 256 << 10) if not orig]
        assert compressed
        for ln, at in compressed:
            assert_host_build_frame(zse, memoryview(blob)[at:at + ln], f"chunk at {at}")


@pytest.fixture(scope="module")
def c4_input_files(c4, tmp_path_factory):
    """The 32 runs as level-0 Parquet files written by the device encoder."""
    schema, _, runs, _ = c4
    d = tmp_path_factory.mktemp("c4_in")
    N.init(0)
    sh = _SchemaHandle(schema, 0)
    metas = []
    try:
        for i, run in enumerate(runs):
            src = SortedRunReader(schema, run)
            try:
                w = KeyValueDataFileWriter(schema, str(d / f"in-{i}.parquet"), 0).write(src._open(sh.handle))
            finally:
                src.close()
            metas.append(w.meta)
    finally:
        sh.close()
    return metas


@pytest.mark.parametrize("file_format", ["orc", "parquet"])
def test_c4_compact_rewriter_at_full_size(c4, c4_input_files, tmp_path, file_format):
    schema, _, _, want = c4
    factory = DeduplicateMergeFunction.factory()
    sections = IntervalPartition(c4_input_files).partition()
    assert len(sections) == 1 and len(sections[0]) == len(c4_input_files)
    rewriter = MergeTreeCompactRewriter(schema, factory, str(tmp_path), options={"file.format": file_format})
    result = rewriter.rewrite_compaction(5, True, sections)
    assert len(result.after) >= 2 and all(m.file_name.endswith("." + file_format) for m in result.after)
    assert sum(m.row_count for m in result.after) == want.n_rows
    got = _read_all(schema, factory, result.after)
    assert got.equals(want), got.first_difference(want)
