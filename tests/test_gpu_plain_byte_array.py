"""PLAIN BYTE_ARRAY pages decoded on the device against pyarrow and against the batch that was written, bit for bit.
The value shapes aim at the staging of the [len][bytes] walk and of the payload copy: values that straddle or exactly
fill 128- and 256-byte windows, values longer than any shared-memory window (300 B, 4 KiB, 70 KiB), empty values,
one-value pages, all-NULL pages, nnz on and off multiples of 32, V1 / V2 pages, Snappy / zstd pages (whose streams
sit at other alignments), PLAIN fallback pages behind a dictionary, runs of several files and the device encoder's
20,000-row pages; and a page whose last length word points past its stream."""
import ctypes as C
import random
import struct

import numpy as np
import pyarrow.parquet as pq
import pytest

from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.format import FileFormat, FormatReaderContext, LocalFileIO, read_section
from paimon_b200.merge_tree_readers import concat_batches
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import arrow_to_batch, write_kv_parquet

pytestmark = pytest.mark.gpu

PG_ERR_FORMAT = 6

SCHEMA = KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("s", "STRING", True),
                                    DataField("b", "BINARY", True), DataField("r", "STRING", False))), ["pk"])

# lengths around 128- and 256-byte windows and beyond them
EDGE_LENGTHS = [0, 1, 3, 4, 5, 15, 16, 17, 120, 123, 124, 125, 127, 128, 129, 131, 255, 256, 300, 508, 509, 512, 513,
                4096, 70 * 1024]


def _text(rng, n):
    return "".join(rng.choice("abcdefghijklmnopqrstuvwxyz0123456789") for _ in range(n))


def _batch(rows):
    return KeyValueBatch.from_rows(SCHEMA, [(k, k + 1, 0, k, s, b, r) for k, (s, b, r) in enumerate(rows)])


def _decode(path):
    rd = FileFormat.from_identifier("parquet").create_reader_factory(SCHEMA).create_reader(
        FormatReaderContext(LocalFileIO(), path))
    try:
        batch = rd.read_batch()
        assert rd.read_batch() is None
        return batch, rd.info()
    finally:
        rd.close()


def _check(batch, path, **opts):
    write_kv_parquet(batch, path, **opts)
    got, info = _decode(path)
    want = arrow_to_batch(SCHEMA, pq.read_table(path))
    assert got.equals(want), got.first_difference(want)
    assert got.equals(batch), got.first_difference(batch)
    return info


def _fetch_and_close(readers):
    out = []
    for r in readers:
        try:
            out.append(r.read_batch())
        finally:
            r.close()
    return out


PLAIN_OPTS = [
    dict(use_dictionary=False),
    dict(use_dictionary=False, data_page_version="2.0"),
    dict(use_dictionary=False, data_page_size=2048),
    dict(use_dictionary=False, compression="snappy"),
    dict(use_dictionary=False, compression="snappy", data_page_version="2.0", data_page_size=4096),
    dict(use_dictionary=False, compression="zstd"),
    dict(use_dictionary=False, compression="zstd", data_page_version="2.0", data_page_size=1000),
]


@pytest.mark.parametrize("opts", PLAIN_OPTS)
def test_value_lengths_around_staging_windows(tmp_path, opts):
    rng = random.Random(11)
    rows = []
    for k in range(3000):
        ln = rng.choice(EDGE_LENGTHS) if rng.random() < 0.3 else rng.randrange(0, 40)
        s = None if rng.random() < 0.3 else _text(rng, ln)
        b = None if rng.random() < 0.2 else bytes(rng.randrange(256) for _ in range(min(ln, 600)))
        rows.append((s, b, _text(rng, rng.choice([0, 7, 128, 133]))))
    _check(_batch(rows), str(tmp_path / "lengths.parquet"), **opts)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 64, 1000, 4096])
def test_null_patterns_and_counts(tmp_path, n):
    """All-NULL pages, pages without NULLs, and every other row NULL (nnz a multiple of 32 or not)."""
    rng = random.Random(n)
    patterns = {
        "all_null": lambda k: None,
        "no_null": lambda k: _text(rng, k % 50),
        "alternate": lambda k: None if k % 2 else _text(rng, k % 37),
        "empty": lambda k: "" if k % 3 else None,
    }
    for name, f in patterns.items():
        rows = [(f(k), None if k % 5 == 0 else bytes([k & 255]) * (k % 9), _text(rng, k % 3)) for k in range(n)]
        for opts in (dict(use_dictionary=False), dict(use_dictionary=False, data_page_version="2.0", data_page_size=256)):
            _check(_batch(rows), str(tmp_path / f"{name}.parquet"), **opts)


def test_one_value_pages(tmp_path):
    rng = random.Random(3)
    rows = [(None if k % 4 == 1 else _text(rng, rng.choice([0, 5, 128, 300])), bytes(k % 7), _text(rng, 1))
            for k in range(200)]
    info = _check(_batch(rows), str(tmp_path / "one.parquet"), use_dictionary=False, data_page_size=1,
                  write_batch_size=1)
    assert info.n_data_pages >= 3 * 200


def test_dictionary_pages_with_plain_fallback(tmp_path):
    """A dictionary that overflows its page limit: the chunk holds dictionary pages, then PLAIN pages."""
    rng = random.Random(5)
    rows = [(_text(rng, rng.randrange(0, 200)), None if k % 3 == 0 else bytes(rng.randrange(256) for _ in range(k % 40)),
             rng.choice(["x", "yy", ""])) for k in range(6000)]
    for opts in (dict(dictionary_pagesize_limit=2048, data_page_size=1024),
                 dict(dictionary_pagesize_limit=4096, data_page_version="2.0", compression="snappy"),
                 dict(dictionary_pagesize_limit=1024, compression="zstd")):
        _check(_batch(rows), str(tmp_path / "fallback.parquet"), **opts)


def test_runs_of_several_files_continue_offsets(tmp_path):
    """Files of one run continue each other's offsets; a run without files is empty."""
    schema = datagen.schema_c3(n_i64=1, n_f64=1, n_str=3)
    opts = [dict(use_dictionary=False), dict(use_dictionary=False, data_page_version="2.0", data_page_size=700),
            dict(use_dictionary=False, compression="snappy", data_page_size=300),
            dict(use_dictionary=False, compression="zstd"), dict(dictionary_pagesize_limit=512, data_page_size=256)]
    run_sizes = [[1237, 1, 3001, 32], [], [5, 64], [4099]]
    files, want, key0, fi = [], [], 0, 0
    for r, sizes in enumerate(run_sizes):
        parts = []
        for n in sizes:
            keys = np.arange(key0, key0 + 2 * n, 2, dtype=np.int64)
            key0 += 2 * n + 10
            part = datagen.make_run(schema, fi, keys, seed=6, null_prob=0.4, str_len=(0, 150))
            path = str(tmp_path / f"f{fi}.parquet")
            write_kv_parquet(part, path, **opts[fi % len(opts)])
            files.append((open(path, "rb").read(), r))
            parts.append(arrow_to_batch(schema, pq.read_table(path)))
            assert parts[-1].equals(part)
            fi += 1
        want.append(concat_batches(schema, parts) if parts else None)
    readers, info = read_section(schema, files, len(run_sizes))
    got = _fetch_and_close(readers)
    for r, (g, w) in enumerate(zip(got, want)):
        if w is None:
            assert g is None or g.n_rows == 0
        else:
            assert g.equals(w), f"run {r}: " + g.first_difference(w)


def test_device_encoded_file_with_20000_row_pages(tmp_path):
    """The bench's files: written by the device encoder (PLAIN, data page V1) with 20,000-row pages."""
    from paimon_b200.compact_rewriter import file_column_names
    from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=4)
    lib = N.init(0)
    sh = _SchemaHandle(schema, 0)
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[nm.encode() for nm in names])
    parts, files, handles, rds = [], [], [], []
    try:
        for i, n in enumerate((65_001, 20_000, 40_032)):
            keys = np.arange(i * 1_000_000, i * 1_000_000 + n, dtype=np.int64)
            part = datagen.make_run(schema, i, keys, seed=8, null_prob=0.5)
            rd = SortedRunReader(schema, part)
            rds.append(rd)
            fh = C.c_uint64(0)
            opts = N.PgParquetWriteOptions(400_000, 20_000)
            N.check(lib.pg_parquet_encode(rd._open(sh.handle), arr, 0, -1, C.byref(opts), C.byref(fh)))
            handles.append(fh.value)
            ptr, size = C.c_void_p(0), C.c_int64(0)
            N.check(lib.pg_parquet_file_device_image(fh.value, C.byref(ptr), C.byref(size)))
            files.append(((ptr.value, size.value), i % 2))
            parts.append((i % 2, part))
            host = np.zeros(size.value, np.uint8)
            N.check(lib.pg_parquet_file_fetch(fh.value, host.ctypes.data, size.value))
            p = str(tmp_path / f"img{i}.parquet")
            host.tofile(p)
            assert arrow_to_batch(schema, pq.read_table(p)).equals(part)
        files_sorted = sorted(files, key=lambda f: f[1])
        readers, _ = read_section(schema, files_sorted, 2)
        got = _fetch_and_close(readers)
        for r in range(2):
            want = concat_batches(schema, [p for rr, p in parts if rr == r])
            assert got[r].equals(want), got[r].first_difference(want)
    finally:
        for h in handles:
            lib.pg_parquet_file_free(h)
        for rd in rds:
            rd.close()
        sh.close()


def test_length_word_past_the_stream_is_a_format_error(tmp_path):
    """The last length word of a PLAIN page points past its stream: the section is refused with PG_ERR_FORMAT (the
    walk checks the bound before it reads), and a good section decoded next on the same device still matches."""
    marker = "LAST-VALUE-OF-THE-PAGE"
    rows = [(f"v{k}", None, "r") for k in range(99)] + [(marker, None, "r")]
    batch = _batch(rows)
    path = str(tmp_path / "bad.parquet")
    write_kv_parquet(batch, path, use_dictionary=False)
    blob = bytearray(open(path, "rb").read())
    needle = struct.pack("<I", len(marker)) + marker.encode()
    at = bytes(blob).find(needle)
    assert at > 0 and bytes(blob).find(needle, at + 1) < 0
    blob[at:at + 4] = struct.pack("<I", len(marker) + 1000)
    with pytest.raises(N.PaimonGpuError) as ei:
        readers, _ = read_section(SCHEMA, [(bytes(blob), 0)], 1)
        _fetch_and_close(readers)
    assert ei.value.status == PG_ERR_FORMAT

    good_path = str(tmp_path / "good.parquet")
    write_kv_parquet(batch, good_path, use_dictionary=False)
    readers, _ = read_section(SCHEMA, [(open(good_path, "rb").read(), 0)], 1)
    got = _fetch_and_close(readers)[0]
    assert got.equals(batch), got.first_difference(batch)
