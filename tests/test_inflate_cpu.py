"""The DEFLATE decoder (paimon_b200/csrc/inflate_device.cuh, RFC 1951 / 1950 / 1952) compiled for the HOST from the same
source the device kernels use, pinned against zlib: stored, fixed and dynamic Huffman blocks, long and overlapping
matches, every compression level, raw / zlib / gzip framing (ORC ZLIB chunks are raw DEFLATE, Parquet GZIP pages are
gzip members)."""
import gzip
import random
import zlib

import numpy as np
import pytest

import codec_filter
from codec_corpora import GZIP, RAW_DEFLATE, ZLIB


@pytest.fixture(scope="module")
def codec(tmp_path_factory):
    return codec_filter.build(str(tmp_path_factory.mktemp("inflate")))


def run(codec, mode, comp: bytes, n: int, cap=None):
    return codec([(mode, comp, n if cap is None else cap)])[0]


def corpus():
    rng = random.Random(1)
    g = np.random.default_rng(1)
    words = ["alpha", "beta", "gamma", "delta", "paimon", "lsm", "merge", "tree", "x", "yy"]
    yield "empty", b""
    yield "one", b"x"
    yield "zeros", bytes(100_000)
    yield "random", g.integers(0, 256, 200_000, dtype=np.uint8).tobytes()
    yield "text", " ".join(rng.choice(words) for _ in range(60_000)).encode()
    yield "sorted_int64", np.arange(0, 150_000, dtype=np.int64).tobytes()
    yield "lowcard", g.integers(0, 7, 300_000, dtype=np.uint8).tobytes()
    yield "skewed", g.geometric(0.3, 300_000).astype(np.uint8).tobytes()
    yield "long_matches", (b"0123456789abcdef" * 5000) + g.integers(0, 256, 1000, dtype=np.uint8).tobytes() + (b"xyz" * 70000)


@pytest.mark.parametrize("level", [0, 1, 6, 9])
def test_decoder_matches_zlib(codec, level):
    for name, data in corpus():
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        raw = co.compress(data) + co.flush()
        r, out = run(codec, RAW_DEFLATE, raw, len(data))
        assert r == len(data) and out == data, f"raw {name} level {level}"
        r, out = run(codec, ZLIB, zlib.compress(data, level), len(data))
        assert r == len(data) and out == data, f"zlib {name} level {level}"
        r, out = run(codec, GZIP, gzip.compress(data, compresslevel=level), len(data))
        assert r == len(data) and out == data, f"gzip {name} level {level}"


def test_fixed_huffman_blocks(codec):
    data = b"abcabcabc hello hello"
    co = zlib.compressobj(9, zlib.DEFLATED, -15, 9, zlib.Z_FIXED)
    raw = co.compress(data) + co.flush()
    r, out = run(codec, RAW_DEFLATE, raw, len(data))
    assert r == len(data) and out == data


def test_malformed_streams_are_rejected(codec):
    data = b"hello hello hello hello " * 100
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    raw = bytearray(co.compress(data) + co.flush())
    assert run(codec, RAW_DEFLATE, bytes(raw), len(data))[0] == len(data)
    assert run(codec, RAW_DEFLATE, bytes(raw), len(data), cap=len(data) - 1)[0] == -1
    assert run(codec, RAW_DEFLATE, bytes(raw[:-4]), len(data))[0] == -1
    rng = random.Random(2)
    for _ in range(300):
        bad = bytearray(raw)
        for _ in range(rng.randrange(1, 4)):
            bad[rng.randrange(len(bad))] = rng.randrange(256)
        r, _ = run(codec, RAW_DEFLATE, bytes(bad), len(data))
        assert r == -1 or 0 <= r <= len(data)
