"""The LZ4 decoder (paimon_b200/csrc/lz4_device.cuh) compiled for the HOST from the same source the device kernels use,
under AddressSanitizer and UBSan, pinned against pyarrow's lz4_raw codec (liblz4's safe decoder): round trips of the
zstd corpus and of the C3 / C5 page bodies, hand-built blocks at every length, offset and end-of-block boundary,
byte-flip and truncation fuzz, and the Hadoop block / chunk framing of Parquet codec 5 pages."""
import os
import random
import struct
import subprocess

import numpy as np
import pyarrow as pa
import pytest

from lz4_parquet import HADOOP_LZ4_CHUNK, lz4_hadoop
from test_zstd_cpu import corpus
from zstd_pages import c3_pages, c5_pages

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RAW, HADOOP = 0, 1


@pytest.fixture(scope="module")
def lz4(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("lz4") / "lz4_host_check")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I" + os.path.join(ROOT, "paimon_b200", "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", "native", "lz4_host_check.cc")])

    def run(records):
        """records: (mode, src bytes, cap) -> [(result, output bytes)]"""
        inp = b"".join(struct.pack("<Bqq", m, cap, len(src)) + bytes(src) for m, src, cap in records)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        p = subprocess.run([exe], input=inp, capture_output=True, env=env)
        assert p.returncode == 0, p.stderr.decode(errors="replace")[-3000:]
        out, pos = [], 0
        for _ in records:
            (r,) = struct.unpack_from("<q", p.stdout, pos)
            pos += 8
            out.append((r, p.stdout[pos:pos + max(r, 0)]))
            pos += max(r, 0)
        assert pos == len(p.stdout)
        return out
    return run


def pyarrow_lz4(block: bytes, size: int):
    """liblz4's safe decoder at the exact size (through pyarrow): the output, or None when it refuses.  pyarrow does
    not report how many bytes liblz4 produced, so only the first ones our decoder reports are comparable."""
    try:
        return pa.decompress(block, decompressed_size=size, codec="lz4_raw", asbytes=True)
    except OSError:
        return None


def compress(data: bytes) -> bytes:
    return pa.compress(data, codec="lz4_raw", asbytes=True)


def test_corpus_and_page_bodies_round_trip(lz4):
    inputs = [d for _, d in corpus()] + c3_pages() + c5_pages()
    res = lz4([(RAW, compress(d), len(d)) for d in inputs])
    for i, (d, (r, out)) in enumerate(zip(inputs, res)):
        assert r == len(d) and out == d, f"input {i}: {r} of {len(d)} bytes"


# ------------------------------------------------------------------ hand-built blocks
#
# liblz4 decodes a sequence on an unchecked shortcut when its literal run is 0..14 bytes, at least 17 input bytes
# follow the token and at least 32 output bytes remain; a match taken there may end anywhere in the output.  The blocks
# whose refusal is pinned below therefore lead with a literal run of 15 or more bytes (or are shorter than 32 bytes),
# so that liblz4 checks them; test_looser_than_liblz4 shows the shortcut itself.

LIT = bytes((i * 37 + 11) & 255 for i in range(70_000))


def varlen(n: int) -> bytes:
    """The length bytes after a nibble of 15: n more, as 255s and a final byte below 255."""
    return b"\xff" * (n // 255) + bytes([n % 255])


def token(lits: int, mlen: int = 4) -> bytes:
    ln, mn = min(lits, 15), min(mlen - 4, 15)
    return bytes([(ln << 4) | mn]) + (varlen(lits - 15) if lits >= 15 else b"")


def seq(lits: bytes, offset: int, mlen: int) -> bytes:
    return token(len(lits), mlen) + lits + struct.pack("<H", offset) + (varlen(mlen - 19) if mlen >= 19 else b"")


def last(lits: bytes) -> bytes:
    return token(len(lits)) + lits


def expand(parts) -> bytes:
    """The output of (literals, offset, match length) sequences and a final literal run."""
    out = bytearray()
    for lits, offset, mlen in parts[:-1]:
        out += lits
        for _ in range(mlen):
            out.append(out[-offset])
    return bytes(out + parts[-1])


def block(parts) -> bytes:
    return b"".join(seq(*p) for p in parts[:-1]) + last(parts[-1])


def boundary_blocks():
    """name -> (block, exact size, expected output or None when refused)"""
    cases = {}
    for n in (14, 15, 15 + 255, 15 + 255 + 1):                 # literal lengths, alone and in front of a match
        cases[f"literals_{n}"] = [LIT[:n]]
        cases[f"literals_{n}_then_match"] = [(LIT[:n], 8, 20), LIT[100:105]]
    for m in (18, 19, 19 + 255):                               # match lengths
        cases[f"match_{m}"] = [(LIT[:15], 8, m), LIT[100:105]]
    for o in list(range(1, 9)) + [65535]:                      # offsets; 1..7 overlap their own output
        cases[f"offset_{o}"] = [(LIT[:max(o, 15)], o, 30), LIT[100:105]]
    cases["offset_past_start"] = [(LIT[:15], 16, 30), LIT[100:105]]
    cases["offset_65535_past_start"] = [(LIT[:65534], 65535, 30), LIT[100:105]]
    for k in (4, 5):                                           # final literal run
        cases[f"last_literals_{k}"] = [(LIT[:15], 15, 16), LIT[100:100 + k]]
    for back, m in ((12, 7), (11, 6)):                         # last match starts 12 / 11 bytes before the end
        cases[f"last_match_at_end_minus_{back}"] = [(LIT[:15], 15, m), LIT[100:105]]
    cases["two_matches"] = [(LIT[:15], 3, 40), (LIT[20:37], 50, 19 + 255 + 3), LIT[100:110]]
    cases["ends_in_a_match"] = None
    out = {}
    for name, parts in cases.items():
        if parts is None:
            b = token(15, 10) + LIT[:15] + struct.pack("<H", 8)
            out[name] = (b, 25, None)
            continue
        valid = all(o <= len(lits) + sum(len(p[0]) + p[2] for p in parts[:i]) for i, (lits, o, _) in enumerate(parts[:-1]))
        exp = expand(parts) if valid else None
        size = len(exp) if exp is not None else sum(len(p[0]) + p[2] for p in parts[:-1]) + len(parts[-1])
        if exp is not None and len(parts) > 1:
            start = len(exp) - len(parts[-1]) - parts[-2][2]   # where the last match starts
            if len(parts[-1]) < 5 or start > len(exp) - 12:
                exp = None
        out[name] = (block(parts), size, exp)
    return out


def test_boundary_blocks_agree_with_liblz4(lz4):
    cases = boundary_blocks()
    res = lz4([(RAW, b, size) for b, size, _ in cases.values()])
    for (name, (b, size, exp)), (r, out) in zip(cases.items(), res):
        ref = pyarrow_lz4(b, size)
        assert (ref is not None) == (exp is not None), f"{name}: the builder and liblz4 disagree"
        if exp is None:
            assert r == -1, f"{name}: accepted, liblz4 refuses"
        else:
            assert r == size and out == exp == ref, f"{name}: {r}"


def test_every_refusal_rule(lz4):
    ok = block([(LIT[:20], 4, 30), LIT[100:106]])
    n = len(expand([(LIT[:20], 4, 30), LIT[100:106]]))
    cases = [
        (RAW, b"", 0, -1),                                     # no input
        (RAW, b"\x00", 0, 0),                                  # the empty block (pyarrow's compress(b"")), cap 0
        (RAW, b"\x0f", 0, -1),                                 # cap 0 takes the one-byte empty block only
        (RAW, b"\x10", 1, -1),                                 # literals past the input
        (RAW, b"\xf0", 100, -1),                               # literal length bytes past the input
        (RAW, b"\xf0\xff\xff", 1000, -1),
        (RAW, last(LIT[:30]), 29, -1),                         # output past cap
        (RAW, last(LIT[:30]), 40, 30),                         # a larger cap is fine
        (RAW, ok, n, n),
        (RAW, ok, n - 1, -1),
        (RAW, ok[:-1], n, -1),                                 # truncated
        (RAW, block([(LIT[:20], 0, 30), LIT[100:106]]), n, -1),      # offset 0
        (RAW, block([(LIT[:20], 21, 30), LIT[100:106]]), n, -1),     # offset before the output
        (RAW, token(20, 30) + LIT[:20] + b"\x04\x00" + b"\xff" * 6, 300, -1),  # match length bytes past the input
    ]
    res = lz4([(m, s, cap) for m, s, cap, _ in cases])
    for i, ((_, s, cap, want), (r, _)) in enumerate(zip(cases, res)):
        assert r == want, f"case {i}: {r} != {want}"


def test_looser_than_liblz4(lz4):
    """Two blocks liblz4's safe decoder takes and this decoder refuses: offset 0 (liblz4 copies from the output
    position itself) and a match that ends the block, taken on liblz4's unchecked shortcut.  Both break the block
    format's rules; every block this decoder accepts liblz4 accepts with the same bytes."""
    off0 = block([(LIT[:8], 0, 8), LIT[100:105]])
    shortcut = token(14, 18) + LIT[:14] + struct.pack("<H", 8) + b"\x00"
    assert pyarrow_lz4(off0, 21) is not None and pyarrow_lz4(shortcut, 32) is not None
    assert [r for r, _ in lz4([(RAW, off0, 21), (RAW, shortcut, 32)])] == [-1, -1]


def test_fuzz_flips_and_truncations(lz4):
    rng = random.Random(7)
    g = np.random.default_rng(7)
    sources = [b"".join(b"%d:%s;" % (i % 97, b"x" * (i % 13)) for i in range(600)),
               g.integers(0, 4, 3000, dtype=np.uint8).tobytes(), bytes(2000) + LIT[:300] + bytes(500)]
    records, expect = [], []
    for data in sources:
        comp = compress(data)
        for _ in range(400):
            bad = bytearray(comp)
            for _ in range(rng.randrange(1, 4)):
                bad[rng.randrange(len(bad))] = rng.randrange(256)
            records.append((RAW, bytes(bad), len(data)))
        for cut in range(1, min(len(comp), 200)):
            records.append((RAW, comp[:-cut], len(data)))
        for cap in (len(data) - 1, len(data) + 1, 0):
            records.append((RAW, comp, cap))
    res = lz4(records)
    accepted = 0
    for (_, src, cap), (r, out) in zip(records, res):
        assert -1 <= r <= cap
        if r >= 0:
            ref = pyarrow_lz4(src, cap) if cap else b""
            assert ref is not None and ref[:r] == out, "accepted a block liblz4 refuses, or decoded it differently"
            accepted += 1
    assert accepted > 0


# ------------------------------------------------------------------ Hadoop framing (Parquet codec 5)

def hadoop_cases():
    g = np.random.default_rng(3)
    text = b"".join(b"row %d value %d;" % (i, i % 101) for i in range(40_000))
    noise = g.integers(0, 256, 600_000, dtype=np.uint8).tobytes()
    return {
        "one_block": [text[:5000]],
        "levels_and_values": [text[:77], text[77:9000]],               # a V1 page: two writes, two blocks
        "chunked_block": [text + noise[:300_000]],                     # 1 block, 3 chunks cut at 261,100 bytes
        "exact_chunk": [noise[:HADOOP_LZ4_CHUNK]],
        "chunk_plus_one": [noise[:HADOOP_LZ4_CHUNK + 1]],
        "blocks_and_chunks": [noise[:10], text[:HADOOP_LZ4_CHUNK * 2 + 5], noise[:600_000]],
        "empty": [],
    }


def test_hadoop_framing_round_trips(lz4):
    cases = hadoop_cases()
    framed = {k: lz4_hadoop(*w) for k, w in cases.items()}
    res = lz4([(HADOOP, framed[k], sum(map(len, w))) for k, w in cases.items()])
    for (name, w), (r, out) in zip(cases.items(), res):
        assert r == sum(map(len, w)) and out == b"".join(w), name
    f = framed["chunked_block"]
    assert struct.unpack(">I", f[:4])[0] == len(cases["chunked_block"][0])
    (c0,) = struct.unpack(">I", f[4:8])
    assert pyarrow_lz4(f[8:8 + c0], HADOOP_LZ4_CHUNK) is not None


def test_hadoop_framing_malformed_lengths_are_refused(lz4):
    a, b = LIT[:3000], bytes(5000)
    good = lz4_hadoop(a, b)
    want = len(a) + len(b)
    blk_a = compress(a)
    chunk_a = struct.pack(">I", len(blk_a)) + blk_a
    rest = good[4 + len(chunk_a):]

    def frame(block_len, chunks, tail=b""):
        return struct.pack(">I", block_len) + chunks + rest + tail
    bad = {
        "want_smaller": (good, want - 1),
        "want_larger": (good, want + 1),
        "block_length_short": (frame(len(a) - 1, chunk_a), want),          # the chunk overruns its block
        "block_length_long": (frame(len(a) + 1, chunk_a), want),           # the block wants another chunk
        "block_past_want": (frame(want + 1, chunk_a), want),
        "chunk_length_past_input": (struct.pack(">I", len(a)) + struct.pack(">I", len(good)) + blk_a, want),
        "chunk_length_short": (frame(len(a), struct.pack(">I", len(blk_a) - 1) + blk_a), want),
        "trailing_bytes": (good + b"\x00\x00\x00", want),
        "trailing_empty_block": (good + b"\x00\x00\x00\x00\x00\x00\x00\x01", want),
        "truncated_block_header": (good[:2], want),
        "truncated_chunk_header": (good[:6], want),
        "truncated": (good[:-1], want),
        "block_without_chunks": (struct.pack(">I", want), want),
    }
    res = lz4([(HADOOP, s, w) for s, w in bad.values()])
    for name, (r, _) in zip(bad, res):
        assert r == -1, name
    # a block of length 0 (Hadoop's end-of-stream mark) holds no chunks
    assert [r for r, _ in lz4([(HADOOP, good, want), (HADOOP, good + b"\x00\x00\x00\x00", want)])] == [want, want]
