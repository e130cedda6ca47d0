"""The carver that lays out the decoders' and the merge's device blocks (device_layout.h), in its host build.  For lists
of regions of several element sizes, zero-count regions included, the sizing pass and the carving pass agree on the
block's bytes, and every region starts on a 256-byte boundary, after the one in front of it, and ends inside the
block."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ELEMS = (1, 2, 3, 4, 8, 24, 32)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = os.path.join(str(tmp_path_factory.mktemp("device_layout")), "device_layout_host_check.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC",
                           "-I" + os.path.join(ROOT, "paimon_b200", "csrc"), "-o", so,
                           os.path.join(ROOT, "tests", "native", "device_layout_host_check.cc")])
    lib = C.CDLL(so)
    lib.layout_check.restype = C.c_int
    lib.layout_check.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def carve(lib, regions):
    """regions: [(element bytes, count)] -> (offsets, sizing-pass bytes, carving-pass bytes)"""
    elem = np.array([e for e, _ in regions] or [1], np.int32)
    count = np.array([n for _, n in regions] or [0], np.int64)
    offsets = np.zeros(max(len(regions), 1), np.int64)
    nbytes = np.zeros(2, np.int64)
    assert lib.layout_check(len(regions), elem.ctypes.data, count.ctypes.data, offsets.ctypes.data,
                            nbytes.ctypes.data) == 0, "the sizing pass returned a non-null pointer"
    return offsets[:len(regions)].tolist(), int(nbytes[0]), int(nbytes[1])


def check(lib, regions):
    offsets, sized, carved = carve(lib, regions)
    assert sized == carved
    end = 0
    for (e, n), off in zip(regions, offsets):
        assert off % 256 == 0, (e, n, off)
        assert off >= end, "regions overlap or come out of order"
        end = off + e * n
        assert end <= carved
    assert end == carved
    return offsets, carved


def test_empty_list(lib):
    assert check(lib, []) == ([], 0)


def test_one_value(lib):
    assert check(lib, [(4, 1)]) == ([0], 4)


def test_offsets_round_each_region_up(lib):
    # 100 bytes, 256 bytes, 1 byte, 3 * 24 bytes: each region starts at the next multiple of 256
    offsets, total = check(lib, [(1, 100), (8, 32), (1, 1), (24, 3)])
    assert offsets == [0, 256, 512, 768]
    assert total == 768 + 72


def test_zero_count_regions(lib):
    # an empty region takes no bytes: it sits where the next region starts, and a trailing one at the block's end
    offsets, total = check(lib, [(8, 0), (4, 10), (32, 0), (32, 0), (2, 5), (3, 0)])
    assert offsets == [0, 0, 256, 256, 256, 512]
    assert total == 512


def test_all_zero(lib):
    assert check(lib, [(8, 0), (1, 0), (24, 0)]) == ([0, 0, 0], 0)


@pytest.mark.parametrize("seed", range(20))
def test_random_lists(lib, seed):
    rnd = random.Random(seed)
    regions = []
    for _ in range(rnd.randint(1, 40)):
        n = rnd.choice([0, 0, 1, rnd.randint(1, 64), rnd.randint(1, 5000), rnd.randint(1, 1 << 20)])
        regions.append((rnd.choice(ELEMS), n))
    check(lib, regions)
