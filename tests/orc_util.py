"""ctypes driver of tests/native/orc_host_check.cc: the HOST build of the ORC decode path (metadata, inflate, stream
decoders — the same sources the device path compiles)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_NP = {1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}


def build(tmp_dir: str, harness: str = "orc_host_check.cc"):
    """harness: orc_host_check.cc (NONE, ZLIB, ZSTD chunks) or orc_lz4_host_check.cc (LZ4 chunks too)"""
    so = os.path.join(tmp_dir, os.path.splitext(harness)[0] + ".so")
    csrc = os.path.join(ROOT, "paimon_b200", "csrc")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I" + csrc, "-o", so,
                           os.path.join(ROOT, "tests", "native", harness), os.path.join(csrc, "orc_meta.cc")])
    lib = C.CDLL(so)
    lib.orc_host_decode.restype = C.c_void_p
    lib.orc_host_decode.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
    lib.orc_host_error.restype = C.c_char_p
    lib.orc_host_rows.restype = C.c_longlong
    lib.orc_host_rows.argtypes = [C.c_void_p]
    lib.orc_host_data.restype = C.c_void_p
    lib.orc_host_data.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_longlong)]
    lib.orc_host_offsets.restype = C.c_void_p
    lib.orc_host_offsets.argtypes = [C.c_void_p, C.c_int]
    lib.orc_host_validity.restype = C.c_void_p
    lib.orc_host_validity.argtypes = [C.c_void_p, C.c_int]
    lib.orc_host_free.argtypes = [C.c_void_p]
    return lib


def decode(lib, file_bytes: bytes, widths):
    """-> (rows, [(values, valid) | (payload, offsets, valid)] per column)"""
    b = np.frombuffer(file_bytes, np.uint8)
    w = np.array(widths, np.int32)
    r = lib.orc_host_decode(b.ctypes.data, len(b), len(widths), w.ctypes.data)
    if not r:
        raise RuntimeError(lib.orc_host_error().decode())
    try:
        n = lib.orc_host_rows(r)
        cols = []
        for c, wd in enumerate(widths):
            nb = C.c_longlong(0)
            dp = lib.orc_host_data(r, c, C.byref(nb))
            data = np.ctypeslib.as_array(C.cast(dp, C.POINTER(C.c_uint8)), (max(nb.value, 1),)).copy()
            val = np.ctypeslib.as_array(C.cast(lib.orc_host_validity(r, c), C.POINTER(C.c_uint32)), ((n + 31) // 32 + 1,)).copy()
            valid = np.unpackbits(val.view(np.uint8), bitorder="little")[:n].astype(bool)
            if wd:
                cols.append((data[: n * wd].view(_NP[wd]), valid))
            else:
                offs = np.ctypeslib.as_array(C.cast(lib.orc_host_offsets(r, c), C.POINTER(C.c_int32)), (n + 1,)).copy()
                cols.append((data, offs, valid))
        return n, cols
    finally:
        lib.orc_host_free(r)
