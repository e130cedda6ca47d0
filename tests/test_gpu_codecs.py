"""The Snappy, zstd and GZIP page decompressors on the device, through the production kernels (k_pq_snappy_lz4,
k_pq_zstd, k_orc_inflate), on the streams test_codecs_cpu.py pins on the host.  Each stream is the values of an INT64
REQUIRED PLAIN page (padded to a multiple of 8 bytes) in a hand-built file (parquet_pages.kv_file):

- Snappy streams at every literal-length and copy boundary, copy-4 elements and long literals, as V1 pages and as V2
  pages behind uncompressed definition levels, one V2 page stored uncompressed;
- zstd and gzip corpora, and sections that mix zstd and gzip pages, more of them than k_pq_zstd has warps, so warps
  decode zstd after gzip after zstd through one shared table slot; some pages' literals take four Huffman streams;
- the fixed list of malformed streams the host build refuses, each alone in a section, refused with PG_ERR_FORMAT,
  and a good section decoded right after on the same device; and corrupt DEFLATE and zstd chunks in ORC streams."""
import struct

import numpy as np
import pytest
import torch

import codec_corpora as K
import orc_stripes as O
import parquet_pages as P
import snappy_streams as S
from paimon_b200 import _native as N
from paimon_b200.format import read_section
from paimon_b200.types import DataField, KeyValueSchema, RowType

pytestmark = pytest.mark.gpu

PG_ERR_FORMAT = 6
CODEC = {K.SNAPPY: P.SNAPPY, K.ZSTD: P.ZSTD, K.GZIP: P.GZIP}


def _schema():
    return KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("v", "BIGINT", True))), ["pk"])


def _v1(stored: bytes, unc: int) -> P.Page:
    n = unc // 8

    def sub(w):
        w.i32(1, n)
        w.i32(2, P.E_PLAIN)
        w.i32(3, P.E_RLE)
        w.i32(4, P.E_RLE)
    return P.Page(P._header(P.DATA_PAGE, unc, len(stored), stored, False, False, 5, sub) + stored, P.DATA_PAGE,
                  P.E_PLAIN, n, unc, len(stored))


def _v2(stored_values: bytes, unc_values: int, compressed: bool = True) -> P.Page:
    """A V2 page of an OPTIONAL column whose rows are all there: uncompressed levels, then the values."""
    n = unc_values // 8
    defs = P.levels([True] * n)
    stored = defs + stored_values

    def sub(w):
        w.i32(1, n)
        w.i32(2, 0)
        w.i32(3, n)
        w.i32(4, P.E_PLAIN)
        w.i32(5, len(defs))
        w.i32(6, 0)
        w.bool(7, compressed)
    unc = len(defs) + unc_values
    return P.Page(P._header(P.DATA_PAGE_V2, unc, len(stored), stored, False, False, 8, sub) + stored, P.DATA_PAGE_V2,
                  P.E_PLAIN, n, unc, len(stored))


def _file(pages, codec: int, optional=False) -> bytes:
    return P.kv_file([sum(p.num_values for p in pages)], [P.ValueColumn("v", P.INT64, optional, [list(pages)],
                                                                         codec=CODEC[codec])])


def _read(files, file_format="parquet"):
    readers, info = read_section(_schema(), [(f, 0) for f in files], 1, file_format=file_format)
    out = []
    for r in readers:
        try:
            out.append(r.read_batch())
        finally:
            r.close()
    return out[0], info


def _check(files, expected: bytes, pages: int):
    batch, info = _read(files)
    want = np.frombuffer(expected, "<i8").tolist()
    got = P.column_values(batch.value_column(1), "BIGINT")
    assert got == want, P.first_mismatch(got, want)
    assert info.n_data_pages == pages + 4 * len(files)          # (the four key columns hold one page per file)


# ------------------------------------------------------------------ Snappy

def _snappy_pages():
    """name -> (stream, padded output) of every writer stream."""
    out = {}
    for name, s in S.streams().items():
        if not s.expected:
            continue
        if len(s.expected) % 8:
            s.literal(S.TEXT[:8 - len(s.expected) % 8])
        out[name] = (s.bytes(), bytes(s.expected))
    return out


SNAPPY_PAGES = _snappy_pages()


@pytest.mark.parametrize("name", sorted(SNAPPY_PAGES))
def test_snappy_pages_v1_and_v2(name):
    stream, want = SNAPPY_PAGES[name]
    _check([_file([_v1(stream, len(want))], K.SNAPPY)], want, 1)
    _check([_file([_v2(stream, len(want))], K.SNAPPY, optional=True)], want, 1)


def test_snappy_section_of_v1_v2_and_uncompressed_v2_pages():
    """V1 pages in a REQUIRED column's file, then V2 pages (one stored uncompressed) in an OPTIONAL column's file."""
    v1 = ["copy4_offsets_past_64k", "literal_61_in_4_length_bytes", "mixed_300k"]
    v2 = ["literal_65537_in_3_length_bytes", "overlap_copy2_offsets_1_to_33"]
    raw = S.TEXT[:4096]
    pages1 = [_v1(SNAPPY_PAGES[k][0], len(SNAPPY_PAGES[k][1])) for k in v1]
    pages2 = [_v2(SNAPPY_PAGES[v2[0]][0], len(SNAPPY_PAGES[v2[0]][1])), _v2(raw, len(raw), compressed=False),
              _v2(SNAPPY_PAGES[v2[1]][0], len(SNAPPY_PAGES[v2[1]][1]))]
    want = b"".join(SNAPPY_PAGES[k][1] for k in v1) + SNAPPY_PAGES[v2[0]][1] + raw + SNAPPY_PAGES[v2[1]][1]
    _check([_file(pages1, K.SNAPPY), _file(pages2, K.SNAPPY, optional=True)], want, len(pages1) + len(pages2))


# ------------------------------------------------------------------ zstd and gzip

def _zstd_gzip_pages():
    """name -> (mode, stream, padded output)"""
    d = K.sample_inputs()
    out = {}
    for name in ("text_600k", "random_300k", "zeros_400k", "rows_300k", "small_text", "padded_counter", "lowcard"):
        data = K.pad8(d[name])
        for level in (1, 19):
            out[f"zstd_{name}_l{level}"] = (K.ZSTD, K.zstd(data, level), data)
        out[f"gzip_{name}"] = (K.GZIP, K.gzip_member(data), data)
    a, b = K.pad8(d["text_600k"][:70_000]), K.pad8(d["rows_300k"][:90_000])
    out["zstd_three_frames"] = (K.ZSTD, K.zstd(a, 3) + K.zstd(b"", 3) + K.zstd(b, 19), a + b)
    out["zstd_skippable_then_frame"] = (K.ZSTD, struct.pack("<II", 0x184D2A53, 5) + b"skip!" + K.zstd(b, 1), b)
    out["gzip_three_members"] = (K.GZIP, K.gzip_member(a, extra=b"xy") + K.gzip_member(b"", name=b"e") +
                                 K.gzip_member(b, level=1, hcrc=True, comment=b"c"), a + b)
    out["gzip_stored_and_fixed"] = (K.GZIP, K.gzip_member(a[:8000], level=0) +
                                    K.gzip_member(b[:8000], name=b"n"), a[:8000] + b[:8000])
    return out


ZG_PAGES = _zstd_gzip_pages()


@pytest.mark.parametrize("name", sorted(ZG_PAGES))
def test_zstd_and_gzip_pages(name):
    mode, stream, want = ZG_PAGES[name]
    _check([_file([_v1(stream, len(want))], mode)], want, 1)


def test_zstd_and_gzip_pages_interleave_on_the_warps():
    """More compressed pages than k_pq_zstd has warps (5 CTAs of 4 warps per SM), in files that alternate zstd and
    gzip, so a warp decodes zstd after gzip after zstd with one table slot; many zstd pages take 4-stream literals."""
    text = K.sample_inputs()["text_600k"]
    rows = K.sample_inputs()["rows_300k"]
    warps = torch.cuda.get_device_properties(0).multi_processor_count * 5 * 4
    n_files, per_file = 40, warps // 20 + 20
    files, want, four = [], b"", 0
    for f in range(n_files):
        mode = K.ZSTD if f % 2 == 0 else K.GZIP
        pages = []
        for i in range(per_file):
            src = text if (f + i) % 3 else rows
            a = ((f * per_file + i) * 977) % (len(src) - 2000)
            data = src[a:a + 8 * (40 + (i * 37) % 200)]
            stream = K.zstd(data, 19 if i % 2 else 3) if mode == K.ZSTD else K.gzip_member(data, level=1 + i % 9)
            if mode == K.ZSTD:
                four += O.zstd_literals_streams(stream) == 4
            pages.append(_v1(stream, len(data)))
            want += data
        files.append(_file(pages, mode))
    assert n_files * per_file > warps and four > n_files, (n_files * per_file, warps, four)
    _check(files, want, n_files * per_file)


# ------------------------------------------------------------------ malformed streams

def _good_section_still_decodes():
    stream, want = SNAPPY_PAGES["mixed_small"]
    _, zs, zwant = ZG_PAGES["zstd_rows_300k_l1"]
    _check([_file([_v1(stream, len(want))], K.SNAPPY), _file([_v1(zs, len(zwant))], K.ZSTD)], want + zwant, 2)


MALFORMED = {f"snappy_{k}": (K.SNAPPY, s, n) for k, (s, n) in S.refusals().items()}
MALFORMED.update(K.malformed_streams())


@pytest.mark.parametrize("name", sorted(MALFORMED))
def test_malformed_stream_is_a_format_error(name):
    mode, stream, n = MALFORMED[name]
    with pytest.raises(N.PaimonGpuError) as ei:
        _read([_file([_v1(stream, n)], mode)])
    assert ei.value.status == PG_ERR_FORMAT, str(ei.value)
    _good_section_still_decodes()


@pytest.mark.parametrize("name", sorted(K.malformed_chunks()))
def test_malformed_orc_chunk_is_a_format_error(name):
    """One compressed chunk of a DATA stream (ZLIB = raw DEFLATE, or zstd) that k_orc_inflate must refuse."""
    mode, body, n = K.malformed_chunks()[name]
    f, _ = O._one("BIGINT", [O.Stream(O.DATA, O.chunk_header(len(body), False) + body, "asis")], 100,
                  codec=O.ZSTD if mode == K.ZSTD else O.ZLIB, block=4096)
    with pytest.raises(N.PaimonGpuError) as ei:
        _read([f.data], file_format="orc")
    assert ei.value.status == PG_ERR_FORMAT, str(ei.value)
    _good_section_still_decodes()
