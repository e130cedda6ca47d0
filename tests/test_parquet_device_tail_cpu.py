"""The Parquet footers of device-resident files, read from byte ranges (pq::read_footers, the path
pg_parquet_read_section takes for PG_MEM_DEVICE files) in the host build, through a reader that records every range it
is asked for.  On pyarrow files of every codec and on multi-row-group files, the parse from ranges equals
parse_footer's, in two rounds of reads, none of them outside its file.  Malformed tails are refused with a format error
before any range leaves the file."""
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


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = os.path.join(str(tmp_path_factory.mktemp("pq_tail")), "parquet_tail_host_check.so")
    csrc = os.path.join(ROOT, "paimon_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + csrc, "-o", so,
                           os.path.join(ROOT, "tests", "native", "parquet_tail_host_check.cc"),
                           os.path.join(csrc, "parquet_meta.cc")])
    lib = C.CDLL(so)
    lib.pq_tail_read.restype = C.c_int
    lib.pq_tail_read.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.pq_tail_error.restype = C.c_char_p
    lib.pq_tail_dump.restype = C.c_char_p
    lib.pq_tail_ranges.restype = C.c_longlong
    lib.pq_tail_ranges.argtypes = [C.POINTER(C.POINTER(C.c_longlong))]
    return lib


def footers(lib, blobs, from_ranges):
    """-> (rounds or None on refusal, dump or error text, recorded ranges [(file, offset, length, round)])"""
    arrs = [np.frombuffer(b, np.uint8) if len(b) else np.zeros(1, np.uint8) for b in blobs]
    ptrs = (C.c_void_p * len(blobs))(*[a.ctypes.data for a in arrs])
    sizes = np.array([len(b) for b in blobs], np.int64)
    rounds = lib.pq_tail_read(ptrs, sizes.ctypes.data, len(blobs), int(from_ranges))
    p = C.POINTER(C.c_longlong)()
    n = lib.pq_tail_ranges(C.byref(p))
    ranges = [tuple(p[4 * i + k] for k in range(4)) for i in range(n)]
    if rounds < 0:
        return None, lib.pq_tail_error().decode(), ranges
    return rounds, lib.pq_tail_dump().decode(), ranges


def assert_inside(blobs, ranges):
    for f, off, n, _ in ranges:
        assert 0 <= off and 0 <= n and off + n <= len(blobs[f]), (f, off, n, len(blobs[f]))


def check_same_parse(lib, blobs):
    rounds, got, ranges = footers(lib, blobs, True)
    assert rounds is not None, got
    _, want, _ = footers(lib, blobs, False)
    assert got == want
    assert rounds == 2
    assert {r for *_, r in ranges} == {0, 1}
    assert_inside(blobs, ranges)
    # round 1: the last 8 bytes of every file; round 2: every footer, right in front of them
    for f, b in enumerate(blobs):
        flen = struct.unpack("<I", b[-8:-4])[0]
        assert (f, len(b) - 8, 8, 0) in ranges
        assert (f, len(b) - 8 - flen, flen, 1) in ranges
    return ranges


def pyarrow_file(n=3000, seed=0, **opts) -> bytes:
    """A flat file of a few types written by pyarrow.parquet."""
    rng = np.random.default_rng(seed)
    t = pa.table({"k": pa.array(np.arange(n, dtype=np.int64)),
                  "v": pa.array(rng.integers(-1000, 1000, n).astype(np.int32)),
                  "s": pa.array([None if i % 7 == 0 else f"s{i % 97}" for i in range(n)]),
                  "d": pa.array(rng.standard_normal(n))})
    buf = io.BytesIO()
    papq.write_table(t, buf, **opts)
    return buf.getvalue()


def with_tail(good: bytes, tail8: bytes) -> bytes:
    return good[:-8] + tail8


@pytest.mark.parametrize("codec", ["none", "snappy", "gzip", "zstd", "lz4"])
def test_pyarrow_files_of_every_codec(lib, codec):
    one = pyarrow_file(3000, seed=1, compression=codec)
    groups = pyarrow_file(20000, seed=2, compression=codec, row_group_size=1500)
    assert papq.ParquetFile(io.BytesIO(groups)).metadata.num_row_groups > 10
    check_same_parse(lib, [one, groups, one])


def test_a_file_without_rows(lib):
    check_same_parse(lib, [pyarrow_file(0)])


def malformed_tails() -> dict:
    good = pyarrow_file(500)
    return {
        "empty": b"",
        "magic_only": b"PAR1PAR1",
        "eleven_bytes": b"PAR1\x00\x00\x00\x00PAR",
        "no_tail_magic": with_tail(good, good[-8:-4] + b"PAR2"),
        "footer_length_past_file": with_tail(good, struct.pack("<I", len(good)) + b"PAR1"),
        "footer_length_one_too_long": with_tail(good, struct.pack("<I", len(good) - 11) + b"PAR1"),
        "footer_length_near_2_32": with_tail(good, struct.pack("<I", 0xFFFFFFF8) + b"PAR1"),
    }


@pytest.mark.parametrize("name", sorted(malformed_tails()))
def test_malformed_tails_are_refused_inside_the_file(lib, name):
    bad = malformed_tails()[name]
    good = pyarrow_file(100, compression="snappy")
    rounds, err, ranges = footers(lib, [good, bad], True)
    assert rounds is None and err.startswith("parquet: "), err
    assert_inside([good, bad], ranges)
    assert footers(lib, [bad], False)[0] is None               # parse_footer refuses the same file
