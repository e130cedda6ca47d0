"""The parse of a section's Parquet footers (pq::parse_footers, which read_footers runs on the footers of
device-resident files) in the host build, against parse_footer run on the files one after another: the same metadata on files of every codec with many row
groups, and, when several footers of a section are malformed, the same error, the first malformed file's in file
order."""
import ctypes as C
import io
import os
import struct
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.parquet as papq
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODECS = ["none", "snappy", "gzip", "zstd", "lz4"]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = os.path.join(str(tmp_path_factory.mktemp("pq_footers")), "parquet_footers_host_check.so")
    csrc = os.path.join(ROOT, "paimon_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I" + csrc,
                           "-I" + os.path.join(ROOT, "tests", "native"), "-o", so,
                           os.path.join(ROOT, "tests", "native", "parquet_footers_host_check.cc"),
                           os.path.join(csrc, "parquet_meta.cc")])
    lib = C.CDLL(so)
    lib.pq_footers_read.restype = C.c_int
    lib.pq_footers_read.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.pq_footers_error.restype = C.c_char_p
    lib.pq_footers_dump.restype = C.c_char_p
    return lib


def parse(lib, blobs, parallel):
    """-> (ok, dump or error text)"""
    arrs = [np.frombuffer(b, np.uint8) for b in blobs]
    ptrs = (C.c_void_p * len(blobs))(*[a.ctypes.data for a in arrs])
    sizes = np.array([len(b) for b in blobs], np.int64)
    if lib.pq_footers_read(ptrs, sizes.ctypes.data, len(blobs), int(parallel)) < 0:
        return False, lib.pq_footers_error().decode()
    return True, lib.pq_footers_dump().decode()


def wide_file(seed, codec, n=6000, n_cols=12, group_rows=400) -> bytes:
    """Many columns and row groups: a footer of tens of KB, like the bench's files."""
    rng = np.random.default_rng(seed)
    cols = {"k": pa.array(np.arange(n, dtype=np.int64))}
    for c in range(n_cols - 1):
        if c % 3 == 0:
            cols[f"s{c}"] = pa.array([None if i % 5 == 0 else f"v{i % 37}" for i in range(n)])
        elif c % 3 == 1:
            cols[f"i{c}"] = pa.array(rng.integers(-9, 9, n).astype(np.int32))
        else:
            cols[f"d{c}"] = pa.array(rng.standard_normal(n))
    buf = io.BytesIO()
    papq.write_table(pa.table(cols), buf, compression=codec, row_group_size=group_rows)
    return buf.getvalue()


def with_footer(good: bytes, footer: bytes) -> bytes:
    flen = struct.unpack("<I", good[-8:-4])[0]
    return good[:-8 - flen] + footer + struct.pack("<I", len(footer)) + b"PAR1"


def footer_of(good: bytes) -> bytes:
    flen = struct.unpack("<I", good[-8:-4])[0]
    return good[-8 - flen:-8]


@pytest.fixture(scope="module")
def files():
    return [wide_file(seed, CODECS[seed % len(CODECS)]) for seed in range(24)]


def test_parallel_parse_equals_the_serial_one(lib, files):
    assert len(footer_of(files[0])) > 16 << 10                   # (footers of the bench's size)
    assert papq.ParquetFile(io.BytesIO(files[0])).metadata.num_row_groups == 15
    ok, want = parse(lib, files, False)
    assert ok, want
    for blobs in (files, files[:1], files[:3], files[::-1]):
        ok, got = parse(lib, blobs, True)
        assert ok, got
        assert got == parse(lib, blobs, False)[1]
    assert parse(lib, files, True)[1] == want


def malformed(good: bytes, kind: str) -> bytes:
    f = footer_of(good)
    if kind == "truncated":
        return with_footer(good, f[: len(f) // 2])
    if kind == "unknown_type":                                    # field 63 of thrift type 13
        return with_footer(good, b"\x0d\x7e" + f)
    if kind == "no_column_meta":                                  # a row group whose one column chunk has no meta_data
        return with_footer(good, b"\x15\x02\x19\x1c\x15\x00\x00\x16\x00\x19\x1c\x19\x1c\x00\x00\x00\x00")
    raise ValueError(kind)


KINDS = ["truncated", "unknown_type", "no_column_meta"]


def test_malformed_footers_alone_are_refused_with_distinct_errors(lib, files):
    errs = []
    for kind in KINDS:
        bad = malformed(files[1], kind)
        ok_s, err_s = parse(lib, [bad], False)
        ok_p, err_p = parse(lib, [bad], True)
        assert not ok_s and not ok_p and err_p == err_s and err_s.startswith("parquet: "), (kind, err_s, err_p)
        errs.append(err_s)
    assert len(set(errs)) == len(KINDS), errs


@pytest.mark.parametrize("order", [(0, 1, 2), (2, 0, 1), (1, 2, 0)])
def test_the_first_malformed_file_in_file_order_is_reported(lib, files, order):
    blobs = list(files)
    for slot, kind_i in zip((5, 11, 19), order):
        blobs[slot] = malformed(files[slot], KINDS[kind_i])
    ok_s, err_s = parse(lib, blobs, False)
    ok_p, err_p = parse(lib, blobs, True)
    assert not ok_s and not ok_p
    assert err_p == err_s == parse(lib, [blobs[5]], False)[1]
