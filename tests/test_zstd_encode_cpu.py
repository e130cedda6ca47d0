"""The Zstandard page encoder (paimon_b200/csrc/zstd_encode_device.cuh) compiled for the HOST from the same source the
device kernels use: every frame decompresses with libzstd (through pyarrow) and with the project's own decoder to
exactly its input, no frame is larger than raw-block framing of its input, and on the lineitem-shaped C5 page bodies
the frames total at most 1.15x libzstd level 1."""
import ctypes as C
import os
import subprocess

import numpy as np
import pyarrow as pa
import pytest

import zstd_pages
from test_zstd_cpu import corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBZSTD = pa.Codec("zstd", compression_level=1)


@pytest.fixture(scope="module")
def zse(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("zse") / "libzse_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "paimon_b200", "csrc"),
                           "-o", so, os.path.join(ROOT, "tests", "native", "zstd_encode_host_check.cc")])
    lib = C.CDLL(so)
    for f in (lib.zse_host_compress, lib.zse_host_decode):
        f.restype = C.c_longlong
        f.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong]
    lib.zse_host_bound.restype = C.c_longlong
    lib.zse_host_bound.argtypes = [C.c_longlong]
    return lib


def compress(lib, data: bytes) -> bytes:
    src = np.frombuffer(data, np.uint8) if data else np.zeros(1, np.uint8)
    cap = lib.zse_host_bound(len(data))
    dst = np.zeros(cap, np.uint8)
    r = lib.zse_host_compress(src.ctypes.data, len(data), dst.ctypes.data, cap)
    assert r > 0
    return dst[:r].tobytes()


def check_frame(lib, data: bytes) -> int:
    frame = compress(lib, data)
    assert LIBZSTD.decompress(frame, decompressed_size=len(data), asbytes=True) == data
    out = np.zeros(len(data) + 64, np.uint8)
    fs = np.frombuffer(frame, np.uint8)
    assert lib.zse_host_decode(fs.ctypes.data, len(frame), out.ctypes.data, len(data)) == len(data)
    assert out[: len(data)].tobytes() == data
    # raw-block framing: frame header (<= 13 bytes with a 1-byte content size... 8) + 3 bytes per 128 KiB block
    header = 6 if len(data) <= 255 else (7 if len(data) <= 65791 else 9)
    assert len(frame) <= header + len(data) + 3 * max(1, -(-len(data) // (128 << 10)))
    assert compress(lib, data) == frame                                # deterministic
    return len(frame)


def test_code_maps_agree_with_the_decoder_tables(zse):
    assert zse.zse_host_check_codes() == 0


def test_decoder_corpus(zse):
    for name, data in corpus():
        check_frame(zse, data)


def test_edges_and_block_types(zse):
    g = np.random.default_rng(3)
    for n in (0, 1, 2, 3, 4, 5, 31, 32, 255, 256, 65791, 65792, 128 << 10, (128 << 10) + 1, 3 * (128 << 10) + 7):
        check_frame(zse, g.integers(0, 4, n, dtype=np.uint8).tobytes())
    assert check_frame(zse, bytes(300_000)) == 9 + 3 * 4               # RLE blocks
    rnd = g.integers(0, 256, 300_000, dtype=np.uint8).tobytes()
    assert check_frame(zse, rnd) == 9 + 300_000 + 3 * 3                # raw blocks
    high = (g.geometric(0.05, 200_000) + 120).clip(0, 255).astype(np.uint8).tobytes()   # byte values >= 128
    assert check_frame(zse, high) < len(high) * 0.8                    # Huffman with FSE-compressed weights


def test_page_images_and_ratio(zse):
    for page in zstd_pages.c3_pages():
        check_frame(zse, page)
    ours = lib1 = 0
    for page in zstd_pages.c5_pages():
        ours += check_frame(zse, page)
        lib1 += len(LIBZSTD.compress(page, asbytes=True))
    print(f"C5 page bodies: host-built frames {ours} B, libzstd-1 {lib1} B, ratio {ours / lib1:.3f}")
    assert ours <= 1.15 * lib1
