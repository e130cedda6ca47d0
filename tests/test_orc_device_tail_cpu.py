"""The ORC file tails of device-resident files, read from byte ranges (orc::read_tails, the path pg_orc_read_section
takes for PG_MEM_DEVICE files) in the host build, through a reader that records every range it is asked for.  On the
reference's golden files, on pyarrow.orc files of every codec the decoder takes and on multi-stripe files in the
device encoder's layout, the parse from ranges equals parse_file's, in at most three rounds of reads, none of them
outside its file.  Malformed tails are refused with a format error before any range leaves the file."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import orc_tails as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "orc")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = os.path.join(str(tmp_path_factory.mktemp("orc_tail")), "orc_tail_host_check.so")
    csrc = os.path.join(ROOT, "paimon_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + csrc, "-o", so,
                           os.path.join(ROOT, "tests", "native", "orc_tail_host_check.cc"), os.path.join(csrc, "orc_meta.cc")])
    lib = C.CDLL(so)
    lib.orc_tail_read.restype = C.c_int
    lib.orc_tail_read.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.orc_tail_error.restype = C.c_char_p
    lib.orc_tail_dump.restype = C.c_char_p
    lib.orc_tail_ranges.restype = C.c_longlong
    lib.orc_tail_ranges.argtypes = [C.POINTER(C.POINTER(C.c_longlong))]
    return lib


def tails(lib, blobs, from_ranges):
    """-> (rounds or None on refusal, dump or error text, recorded ranges [(file, offset, length, round)])"""
    arrs = [np.frombuffer(b, np.uint8) if len(b) else np.zeros(1, np.uint8) for b in blobs]
    ptrs = (C.c_void_p * len(blobs))(*[a.ctypes.data for a in arrs])
    sizes = np.array([len(b) for b in blobs], np.int64)
    rounds = lib.orc_tail_read(ptrs, sizes.ctypes.data, len(blobs), int(from_ranges))
    p = C.POINTER(C.c_longlong)()
    n = lib.orc_tail_ranges(C.byref(p))
    ranges = [tuple(p[4 * i + k] for k in range(4)) for i in range(n)]
    if rounds < 0:
        return None, lib.orc_tail_error().decode(), ranges
    return rounds, lib.orc_tail_dump().decode(), ranges


def assert_inside(blobs, ranges):
    for f, off, n, _ in ranges:
        assert 0 <= off and 0 <= n and off + n <= len(blobs[f]), (f, off, n, len(blobs[f]))


def check_same_parse(lib, blobs):
    rounds, got, ranges = tails(lib, blobs, True)
    assert rounds is not None, got
    _, want, _ = tails(lib, blobs, False)
    assert got == want
    assert 1 <= rounds <= 3
    assert {r for *_, r in ranges} == set(range(rounds))
    assert_inside(blobs, ranges)
    return rounds, ranges


def encoder_file(tmp_path_factory, n, stripe_rows, codec):
    """A file written by the host build of the device encoder (orc_encode_host_check.cc: its stripe and tail layout)."""
    import test_orc_encode_cpu as E
    d = str(tmp_path_factory.mktemp("orc_tail_enc"))
    so = os.path.join(d, "liborc_enc_host.so")
    csrc = os.path.join(ROOT, "paimon_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + csrc, "-o", so,
                           os.path.join(ROOT, "tests", "native", "orc_encode_host_check.cc"), os.path.join(csrc, "orc_meta.cc")])
    enc = C.CDLL(so)
    enc.orc_enc_host_write.restype = C.c_longlong
    enc.orc_enc_host_write.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_longlong, C.c_longlong, C.c_int, C.c_longlong]
    enc.orc_enc_host_bytes.restype = C.POINTER(C.c_uint8)
    enc.orc_enc_host_error.restype = C.c_char_p
    return E.write(enc, E.make_columns(n, 0.2, seed=n), n, stripe_rows, codec=codec)


def test_golden_files(lib):
    blobs = [open(os.path.join(GOLDEN, f), "rb").read() for f in sorted(os.listdir(GOLDEN)) if f.endswith(".orc")]
    assert len(blobs) == 2
    for b in blobs:
        check_same_parse(lib, [b])
    check_same_parse(lib, blobs)


@pytest.mark.parametrize("codec", ["uncompressed", "zlib", "lz4", "zstd"])
def test_pyarrow_files_of_every_codec(lib, codec):
    one = T.pyarrow_file(3000, seed=1, compression=codec)
    striped = T.pyarrow_file(20000, seed=2, compression=codec, stripe_size=4096, compression_block_size=65536)
    rounds, _ = check_same_parse(lib, [one, striped, one])
    assert rounds == 2 or rounds == 3


@pytest.mark.parametrize("codec", [0, 5], ids=["none", "zstd"])
def test_encoder_layout_with_footers_beyond_the_first_read(lib, tmp_path_factory, codec):
    """Thousands of stripes: the Footer is larger than the 16 KiB first read, so a second round fetches the rest of it
    (only for that file), and all stripe footers of every file come in the third."""
    big = encoder_file(tmp_path_factory, 48000, 4, codec)
    small = encoder_file(tmp_path_factory, 700, 256, codec)
    rounds, ranges = check_same_parse(lib, [small, big, small])
    assert rounds == 3
    assert {f for f, *_, r in ranges if r == 1} == {1}


def test_a_file_smaller_than_the_first_read(lib):
    b = T.pyarrow_file(5, compression="zstd")
    assert len(b) < 16384
    rounds, ranges = check_same_parse(lib, [b])
    assert rounds == 2
    assert (0, 0, len(b), 0) in ranges


@pytest.mark.parametrize("name", sorted(T.malformed_tails()))
def test_malformed_tails_are_refused_inside_the_file(lib, name):
    bad = T.malformed_tails()[name]
    good = T.pyarrow_file(100, compression="zlib")
    rounds, err, ranges = tails(lib, [good, bad], True)
    assert rounds is None and err.startswith("orc: ") and "is not decoded" not in err, err
    assert_inside([good, bad], ranges)
    assert tails(lib, [bad], False)[0] is None                 # parse_file refuses the same file
