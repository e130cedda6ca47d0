"""The Zstandard page decoder (paimon_b200/csrc/zstd_device.cuh, RFC 8878) compiled for the HOST from the same source
the device kernel uses, pinned against libzstd (through pyarrow): every block type, Huffman literals (1 and 4 streams,
FSE-compressed and direct weights, treeless), predefined / RLE / FSE / repeat sequence tables, repeat offsets, long
and overlapping matches, multi-block frames, levels 1..19.  zstd-jni (the reference's codec) wraps the same libzstd."""
import random

import numpy as np
import pyarrow as pa
import pytest

import codec_filter
from codec_corpora import ZSTD


@pytest.fixture(scope="module")
def zs(tmp_path_factory):
    return codec_filter.build(str(tmp_path_factory.mktemp("zs")))


def roundtrip(codec, data: bytes, level: int) -> bool:
    comp = pa.Codec("zstd", compression_level=level).compress(data, asbytes=True)
    [(r, out)] = codec([(ZSTD, comp, len(data))])
    return r == len(data) and out == data


def corpus():
    rng = random.Random(1)
    g = np.random.default_rng(1)
    words = ["alpha", "beta", "gamma", "delta", "paimon", "lsm", "merge", "tree", "x", "yy"]
    yield "empty", b""
    yield "one", b"x"
    yield "zeros", bytes(100_000)
    yield "random", g.integers(0, 256, 300_000, dtype=np.uint8).tobytes()
    yield "text", " ".join(rng.choice(words) for _ in range(60_000)).encode()
    yield "sorted_int64", np.arange(0, 200_000, dtype=np.int64).tobytes()
    yield "lowcard", g.integers(0, 7, 500_000, dtype=np.uint8).tobytes()
    yield "skewed", g.geometric(0.3, 400_000).astype(np.uint8).tobytes()
    yield "doubles", (g.integers(0, 1000, 100_000) / 8.0).astype(np.float64).tobytes()
    yield "multi_block", g.integers(0, 50, 1_500_000, dtype=np.uint8).tobytes()
    yield "long_matches", (b"0123456789abcdef" * 5000) + g.integers(0, 256, 1000, dtype=np.uint8).tobytes() + (b"xyz" * 70000)
    # a Parquet-like page: RLE/bit-packed dictionary ids + plain strings
    yield "page_like", b"".join((b"%08d" % (i % 977)) + b"user_" + (b"%07d" % i) for i in range(40_000))


@pytest.mark.parametrize("level", [1, 3, 9, 19])
def test_decoder_matches_libzstd(zs, level):
    for name, data in corpus():
        assert roundtrip(zs, data, level), f"{name} at level {level}"


def test_malformed_streams_are_rejected(zs):
    data = b"hello hello hello hello " * 100
    comp = bytearray(pa.Codec("zstd", compression_level=3).compress(data, asbytes=True))

    def run(buf, cap):
        return zs([(ZSTD, bytes(buf), cap)])[0][0]
    assert run(comp, len(data)) == len(data)
    assert run(comp, len(data) - 1) == -1                     # does not fit
    assert run(comp[:-3], len(data)) == -1                    # truncated
    bad = bytearray(comp); bad[0] ^= 0xFF
    assert run(bad, len(data)) == -1                          # magic
    rng = random.Random(2)
    for _ in range(300):                                      # random corruption never runs out of bounds
        bad = bytearray(comp)
        for _ in range(rng.randrange(1, 4)):
            bad[rng.randrange(4, len(bad))] = rng.randrange(256)
        r = run(bad, len(data))
        assert r == -1 or 0 <= r <= len(data)
