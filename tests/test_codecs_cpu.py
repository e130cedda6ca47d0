"""The Snappy, zstd and DEFLATE page decompressors (snappy_device.cuh, zstd_device.cuh, inflate_device.cuh) compiled for
the HOST from the same sources the device kernels use, under AddressSanitizer and UBSan, with every buffer allocated
at its exact size (tests/native/codec_host_check.cc, run through codec_filter.py).

- Snappy: hand-built streams (snappy_streams.py) at every literal-length and copy boundary, decoded equal to the
  writer and to libsnappy; one malformed stream per refusal rule.
- zstd, raw DEFLATE, zlib and gzip: corpora that cover the block, literal and header kinds, decoded equal to libzstd
  and zlib.
- Seeded byte-flip and truncation fuzz for all four codecs: every stream a decoder accepts, the reference library
  accepts with the same bytes.
- The checks the decoders skip (gzip CRC32 and header CRC16, zlib Adler-32, zstd content checksum), compared with the
  reference with the check off, and the gzip ISIZE, which is checked."""
import gzip
import random
import struct
import zlib

import pytest

import codec_corpora as K
import codec_filter
import snappy_streams as S
from codec_corpora import GZIP, RAW_DEFLATE, SNAPPY, ZLIB, ZSTD, reference


@pytest.fixture(scope="module")
def codec(tmp_path_factory):
    return codec_filter.build(str(tmp_path_factory.mktemp("codecs")))


# ------------------------------------------------------------------ Snappy

def test_snappy_streams_match_the_writer_and_libsnappy(codec):
    cases = S.streams()
    res = codec([(SNAPPY, s.bytes(), len(s.expected)) for s in cases.values()])
    for (name, s), (r, out) in zip(cases.items(), res):
        want = bytes(s.expected)
        assert S.libsnappy(s.bytes(), len(want)) == want, f"{name}: the writer and libsnappy disagree"
        assert r == len(want) and out == want, f"{name}: {r} of {len(want)} bytes"
    src, want = S.non_canonical_preamble()
    assert S.libsnappy(src, len(want)) == want
    assert codec([(SNAPPY, src, len(want))]) == [(len(want), want)]


def test_snappy_streams_from_libsnappy(codec):
    inputs = list(K.sample_inputs().values()) + [b""]
    res = codec([(SNAPPY, S.compress(d), len(d)) for d in inputs])
    for d, (r, out) in zip(inputs, res):
        assert r == len(d) and out == d


def test_snappy_refusals(codec):
    cases = S.refusals()
    res = codec([(SNAPPY, src, n) for src, n in cases.values()])
    for (name, (src, n)), (r, _) in zip(cases.items(), res):
        assert S.libsnappy(src, n) is None, f"{name}: libsnappy takes it"
        assert r == -1, f"{name}: accepted ({r})"
    good = S.streams()["mixed_small"]
    n = len(good.expected)
    assert [r for r, _ in codec([(SNAPPY, good.bytes(), n - 1), (SNAPPY, good.bytes(), n + 1)])] == [-1, -1]


def test_snappy_refusal_controls(codec):
    """Each refusal whose fault is one field, with only that field corrected, decodes to its size: the stream is
    refused for that field and nothing else."""
    cases = S.refusal_controls()
    refused = S.refusals()
    res = codec([(SNAPPY, src, len(want)) for src, want in cases.values()])
    for (name, (src, want)), (r, out) in zip(cases.items(), res):
        assert len(src) == len(refused[name][0]) and len(want) == refused[name][1], name
        assert S.libsnappy(src, len(want)) == want, f"{name}: libsnappy refuses the control"
        assert r == len(want) and out == want, f"{name}: the control is refused ({r})"


# ------------------------------------------------------------------ zstd and DEFLATE corpora

def test_zstd_corpus_matches_libzstd(codec):
    cases = K.zstd_corpus()
    kinds = set()
    res = codec([(ZSTD, s, len(d)) for s, d in cases.values()])
    for (name, (s, d)), (r, out) in zip(cases.items(), res):
        assert K.libzstd(s, len(d)) == d, name
        assert r == len(d) and out == d, f"{name}: {r} of {len(d)} bytes"
        kinds |= K.zstd_kinds(s)
    assert kinds >= {"multi_block_frame", "raw_block", "rle_block", "compressed_block", "raw_literals", "rle_literals",
                     "huffman_1_stream", "huffman_4_streams", "treeless_1_stream", "treeless_4_streams",
                     "skippable_frame"}, kinds


@pytest.mark.parametrize("mode", [RAW_DEFLATE, ZLIB, GZIP])
def test_deflate_corpora_match_zlib(codec, mode):
    cases = K.gzip_corpus() if mode == GZIP else K.deflate_corpus(-15 if mode == RAW_DEFLATE else 15)
    res = codec([(mode, s, len(d)) for s, d in cases.values()])
    for (name, (s, d)), (r, out) in zip(cases.items(), res):
        assert reference(mode, s, len(d)) == d, f"{name}: zlib reads something else"
        assert r == len(d) and out == d, f"{name}: {r} of {len(d)} bytes"
    if mode == GZIP:
        for name in ("fextra", "fname", "fcomment", "fhcrc", "three_members"):
            assert gzip.decompress(cases[name][0]) == cases[name][1]     # and they are valid with every CRC checked


# ------------------------------------------------------------------ fuzz

def _fuzz_sources(mode):
    d = K.sample_inputs()
    texts = [d["text_600k"][:4000], d["rows_300k"][:6000], d["lowcard"][:3000], d["small_text"]]
    if mode == SNAPPY:
        return [(S.compress(t), t) for t in texts] + \
               [(s.bytes(), bytes(s.expected)) for s in (S.streams()["mixed_small"], S.streams()["copy1_lengths_4_to_11"])]
    if mode == ZSTD:
        return [(K.zstd(t, lv), t) for t, lv in zip(texts, (1, 3, 19, 3))] + \
               [(K.zstd(texts[0], 3) + K.zstd(texts[3], 19), texts[0] + texts[3])]
    if mode == GZIP:
        return [(K.gzip_member(t), t) for t in texts] + \
               [(K.gzip_member(texts[3], extra=b"xy", name=b"n", comment=b"c", hcrc=True) + K.gzip_member(texts[2], level=0),
                 texts[3] + texts[2])]
    wbits = -15 if mode == RAW_DEFLATE else 15
    return [(K.deflate(t, 6, st, wbits), t) for t, st in zip(texts, (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED,
                                                                      zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE))] + \
           [(K.deflate(texts[1][:2000], 0, wbits=wbits), texts[1][:2000])]


@pytest.mark.parametrize("mode", [SNAPPY, ZSTD, RAW_DEFLATE, ZLIB, GZIP])
def test_fuzz_flips_and_truncations(codec, mode):
    rng = random.Random(11 + mode)
    records = []
    for comp, data in _fuzz_sources(mode):
        for _ in range(700):
            bad = bytearray(comp)
            for _ in range(rng.randrange(1, 4)):
                bad[rng.randrange(len(bad))] = rng.randrange(256)
            records.append((mode, bytes(bad), len(data)))
        for cut in sorted(rng.sample(range(1, len(comp)), min(len(comp) - 1, 150))):
            records.append((mode, comp[:-cut], len(data)))
        for cap in (len(data) - 1, len(data) + 1):
            records.append((mode, comp, cap))
    res = codec(records)
    accepted = refused = 0
    for (_, src, cap), (r, out) in zip(records, res):
        assert -1 <= r <= cap
        if r < 0:
            refused += 1
            continue
        accepted += 1
        assert reference(mode, src, r) == out, "accepted a stream the reference refuses, or decoded it differently"
    assert accepted > 0 and refused > 0 and len(records) > 2000


# ------------------------------------------------------------------ the checks the decoders skip, and gzip ISIZE

def test_looser_than_the_references(codec):
    """The decoders skip the gzip CRC32 and header CRC16, the zlib Adler-32 and the zstd content checksum.  Streams
    whose only fault is one of these are accepted, with the bytes the reference produces once the check is off.  For
    gzip and zlib that is reference(), which recomputes the CRCs before zlib reads the stream.  libzstd cannot be told
    to skip the content checksum (pyarrow has no such option), so the zstd case is compared with libzstd's reading of
    the same frame without the checksum flag and bytes."""
    data = K.sample_inputs()["rows_300k"][:20_000]
    good_gz = K.gzip_member(data, name=b"n", hcrc=True)
    bad_crc = good_gz[:-8] + struct.pack("<I", zlib.crc32(data) ^ 1) + good_gz[-4:]
    h = 10 + 2
    bad_hcrc = good_gz[:h] + bytes([good_gz[h] ^ 1]) + good_gz[h + 1:]
    good_z = K.deflate(data, 6, wbits=15)
    bad_adler = good_z[:-4] + struct.pack(">I", zlib.adler32(data) ^ 1)
    frame = K.zstd(data, 3)
    with_checksum = frame[:4] + bytes([frame[4] | 4]) + frame[5:] + b"\x00\x11\x22\x33"
    for s in (bad_crc, bad_hcrc):
        with pytest.raises(zlib.error):
            zlib.decompress(s, 31)
    with pytest.raises(zlib.error):
        zlib.decompress(bad_adler, 15)
    assert K.libzstd(with_checksum, len(data)) is None and K.libzstd(frame, len(data)) == data
    cases = [(GZIP, bad_crc), (GZIP, bad_hcrc), (ZLIB, bad_adler), (ZSTD, with_checksum)]
    res = codec([(m, s, len(data)) for m, s in cases])
    for (m, s), (r, out) in zip(cases, res):
        assert r == len(data) and out == data
        if m != ZSTD:
            assert reference(m, s, len(data)) == data


def test_gzip_isize_is_checked(codec):
    data = K.sample_inputs()["text_600k"][:9000]
    good = K.gzip_member(data)
    wrong = [good[:-4] + struct.pack("<I", len(data) + d) for d in (1, -1, 1 << 16)]
    two = K.gzip_member(data) + wrong[0]
    for s in wrong + [two]:
        with pytest.raises(zlib.error):
            d = zlib.decompressobj(31)
            d.decompress(s)
            if d.unused_data:
                zlib.decompressobj(31).decompress(d.unused_data)
    for s, n in [(w, len(data)) for w in wrong] + [(two, 2 * len(data))]:
        assert reference(GZIP, s, n) is None
        assert reference(GZIP, s, n - 8) is None and reference(GZIP, s, n + 8) is None
    assert reference(GZIP, good, len(data)) == data
    res = codec([(GZIP, good, len(data))] + [(GZIP, s, len(data)) for s in wrong] + [(GZIP, two, 2 * len(data))])
    assert [r for r, _ in res] == [len(data), -1, -1, -1, -1]


def test_malformed_zstd_and_gzip_streams_are_refused(codec):
    """The fixed lists of malformed streams and ORC chunk bodies the device tests also give the production kernels."""
    cases = {**K.malformed_streams(), **{"chunk_" + k: v for k, v in K.malformed_chunks().items()}}
    res = codec([(m, s, n) for m, s, n in cases.values()])
    for (name, (m, s, n)), (r, _) in zip(cases.items(), res):
        assert reference(m, s, n) is None, f"{name}: the reference takes it"
        assert r == -1, f"{name}: accepted ({r})"
