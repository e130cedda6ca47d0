"""pg_orc_read_section on file bytes already in device memory (PG_MEM_DEVICE descriptors): the tails come back through
small reads, the compression chunks are walked on the device, and the bytes are read in place.  Every comparison is bit
for bit over values, offsets and validity against the decode of the same files from host bytes:
  * the all-types files of test_gpu_orc.py under NONE / ZLIB / LZ4 / ZSTD and RLE v1 / v2, one file per section and
    runs mixing host and device descriptors, with and without a read-type projection;
  * the hand-built stripes of orc_stripes.py: the same runs, or the same PG_ERR_FORMAT;
  * pg_orc_encode output read in place through pg_parquet_file_device_image, against the source batch;
  * ORC files sent through FileUpload with two uploads in flight.
Device files sit inside larger buffers filled with poison bytes, so that a read outside a file changes the result
instead of faulting; malformed tails placed that way are refused with PG_ERR_FORMAT."""
import ctypes as C

import numpy as np
import pyarrow.orc as orc
import pytest
import torch

import orc_stripes as S
import orc_tails as T
import parquet_pages as P
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import is_varlen, unpack_validity
from paimon_b200.compact_rewriter import KeyValueDataFileWriter
from paimon_b200.format import FileUpload, read_section
from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, RowType
from parquet_util import to_arrow
from test_gpu_orc import all_types_schema, random_batch, write_kv_orc

pytestmark = pytest.mark.gpu

PG_ERR_FORMAT = 6
PAD = 4096


class DeviceFiles:
    """Files copied into device buffers between PAD poison bytes on each side; keeps the buffers alive."""

    def __init__(self):
        self.bufs = []

    def __call__(self, blob: bytes):
        buf = torch.full((PAD + len(blob) + PAD,), 0xA5, dtype=torch.uint8, device="cuda")
        if blob:
            buf[PAD:PAD + len(blob)] = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
        torch.cuda.synchronize()
        self.bufs.append(buf)
        return (buf.data_ptr() + PAD, len(blob))


def decode(schema, files, n_runs, **kw):
    readers, info = read_section(schema, files, n_runs, file_format="orc", **kw)
    out = []
    for r in readers:
        try:
            out.append(r.read_batch())
        finally:
            r.close()
    return out, info


def assert_same(got, want):
    """Bit for bit: validity, values (every slot, NULL ones included), offsets and payload."""
    assert got.n_rows == want.n_rows
    n = got.n_rows
    for ci, (a, b) in enumerate(zip(got.columns, want.columns)):
        assert (a is None) == (b is None), ci
        if a is None:
            continue
        assert np.array_equal(unpack_validity(a.valid, n), unpack_validity(b.valid, n)), ci
        if is_varlen(a.type):
            oa, ob = np.asarray(a.offsets[:n + 1]), np.asarray(b.offsets[:n + 1])
            assert np.array_equal(oa, ob), ci
            assert np.asarray(a.data[:oa[-1]]).tobytes() == np.asarray(b.data[:ob[-1]]).tobytes(), ci
        else:
            assert np.asarray(a.data[:n]).tobytes() == np.asarray(b.data[:n]).tobytes(), ci


def assert_runs_same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if w is None or g is None:
            assert g is None and w is None
        else:
            assert_same(g, w)


CODECS = ["uncompressed", "zlib", "lz4", "zstd"]


@pytest.mark.parametrize("rle", ["0.11", "0.12"], ids=["rle_v1", "rle_v2"])
@pytest.mark.parametrize("codec", CODECS)
def test_all_types_from_device_bytes(tmp_path, codec, rle):
    schema = all_types_schema()
    dev = DeviceFiles()
    blobs = []
    for n, null_p in ((1, 0.0), (33, 0.3), (5000, 0.25), (12000, 0.9)):
        path = str(tmp_path / f"a{n}.orc")
        write_kv_orc(random_batch(schema, n, seed=n + 5, null_p=null_p), path, compression=codec, file_version=rle,
                     stripe_size=64 * 1024)
        blob = open(path, "rb").read()
        blobs.append(blob)
        want, _ = decode(schema, [(blob, 0)], 1)
        got, info = decode(schema, [(dev(blob), 0)], 1)
        assert_runs_same(got, want)
        assert info.file_bytes == len(blob)
    # runs of several files, host and device descriptors mixed, whole and projected
    files_h = [(b, i % 3) for i, b in enumerate(blobs + blobs[:2])]
    files_h.sort(key=lambda f: f[1])
    files_m = [(dev(b) if i % 2 else b, r) for i, (b, r) in enumerate(files_h)]
    for mask in (None, [f.name in ("pk", "l", "low", "dt") for f in schema.value_type.fields]):
        want, _ = decode(schema, files_h, 3, read_value_fields=mask)
        got, info = decode(schema, files_m, 3, read_value_fields=mask)
        assert_runs_same(got, want)
        assert info.n_files == len(files_h)


def _stripe_schema(vtype):
    return KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("v", vtype, True))), ["pk"])


def _host_or_error(schema, files):
    try:
        return decode(schema, files, 1)[0], None
    except N.PaimonGpuError as e:
        return None, e.status


@pytest.mark.parametrize("name", sorted(S.well_formed_cases()) + sorted(S.malformed_cases()))
def test_hand_built_stripes_from_device_bytes(name):
    if name in S.well_formed_cases():
        case = S.well_formed_cases()[name]()
        files, vtype = case.files, case.vtype
    else:
        f, vtype = S.malformed_cases()[name]()
        files = [f]
    schema = _stripe_schema(S.VTYPES[vtype].read)
    dev = DeviceFiles()
    want, want_st = _host_or_error(schema, [(f.data, 0) for f in files])
    got, got_st = _host_or_error(schema, [(dev(f.data), 0) for f in files])
    assert got_st == want_st
    if want_st is None:
        assert_runs_same(got, want)
    else:
        assert want_st == PG_ERR_FORMAT
        good = S.validity_join_case()                   # the device decodes a good section right after
        sch = _stripe_schema(S.VTYPES[good.vtype].read)
        batch = decode(sch, [(dev(f.data), 0) for f in good.files], 1)[0][0]
        assert P.column_values(batch.value_column(1), S.VTYPES[good.vtype].read) == good.expected


@pytest.mark.parametrize("compression", ["none", "zstd"])
def test_encoder_output_read_in_place(compression):
    """pg_orc_encode -> pg_parquet_file_device_image -> pg_orc_read_section(PG_MEM_DEVICE): the file the device just
    wrote is read without a trip through the host, and equals the source batch."""
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=2)
    batch = datagen.make_run(schema, 0, np.arange(0, 90_000, 3, dtype=np.int64), seed=4, null_prob=0.3)
    lib = N.init(0)
    sh = _SchemaHandle(schema, 0)
    rd = SortedRunReader(schema, batch)
    w = KeyValueDataFileWriter(schema, "unused.orc", level=0, file_format="orc", compression=compression,
                               stripe_rows=7000)
    names = [f.name for f in schema.file_fields()]
    arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
    fh = C.c_uint64(0)
    try:
        N.check(lib.pg_orc_encode(rd._open(sh.handle), arr, 0, -1, C.byref(w.orc_opts), C.byref(fh)))
        try:
            ptr, size = C.c_void_p(0), C.c_int64(0)
            N.check(lib.pg_parquet_file_device_image(fh.value, C.byref(ptr), C.byref(size)))
            (got,), info = decode(schema, [((ptr.value, size.value), 0)], 1)
            host = np.empty(size.value, np.uint8)
            N.check(lib.pg_parquet_file_fetch(fh.value, host.ctypes.data, size.value))
        finally:
            N.check(lib.pg_parquet_file_free(fh.value))
    finally:
        rd.close()
        sh.close()
    assert got.equals(batch), got.first_difference(batch)
    assert info.n_chunks == schema.n_cols * 5                # 30,000 rows in stripes of 7,000
    (want,), _ = decode(schema, [(host.tobytes(), 0)], 1)
    assert_same(got, want)


def test_sections_through_file_upload(tmp_path):
    """Two uploads in flight, consumed in order: the descriptors wait() hands back decode to the host decode's runs."""
    schema = datagen.schema_c3(n_i64=2, n_f64=1, n_str=2)
    files = []
    for i, n in enumerate((3001, 17, 1200, 9000)):
        keys = np.arange(i * 100_000, i * 100_000 + n, dtype=np.int64)
        part = datagen.make_run(schema, i, keys, seed=9, null_prob=0.4, delete_prob=0.1)
        path = str(tmp_path / f"u{i}.orc")
        orc.write_table(to_arrow(part), path, compression=CODECS[i])
        files.append((open(path, "rb").read(), i % 2))
    files.sort(key=lambda f: f[1])
    want, _ = decode(schema, files, 2)
    uploads = [FileUpload(files), FileUpload(files)]
    try:
        for up in uploads:
            got, _ = decode(schema, up.wait(), 2)
            assert_runs_same(got, want)
    finally:
        for up in uploads:
            up.close()


@pytest.mark.parametrize("name", sorted(T.malformed_tails()))
def test_malformed_tails_in_device_memory_are_format_errors(name):
    schema = all_types_schema()
    dev = DeviceFiles()
    bad = T.malformed_tails()[name]
    good = T.pyarrow_file(50, compression="zlib")
    with pytest.raises(N.PaimonGpuError) as ei:
        read_section(schema, [(dev(good), 0), (dev(bad), 0)], 1, file_format="orc", check_names=False)
    assert ei.value.status == PG_ERR_FORMAT, str(ei.value)
    case = S.validity_join_case()
    sch = _stripe_schema(S.VTYPES[case.vtype].read)
    batch = decode(sch, [(dev(f.data), 0) for f in case.files], 1)[0][0]
    assert P.column_values(batch.value_column(1), S.VTYPES[case.vtype].read) == case.expected
