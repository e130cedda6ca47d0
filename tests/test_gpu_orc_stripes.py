"""The device ORC decoder on hand-built stripes (orc_stripes.py), compared with the builder's values (integers
exactly, floats by bit pattern, strings by bytes, validity bit for bit) and with pyarrow.orc's reading of the same
files: every RLE v2 sub-encoding at its header-field edges, RLE v1, byte RLE and boolean streams, DECIMAL per-value
scales, DIRECT and DICTIONARY strings, compression chunks under ZLIB, ZSTD and LZ4.  A run of files whose stripes of 1
to 4,095 rows share validity words; a section of more streams than the stream decode has warps, so warps decode
several streams of different codecs.  Malformed streams and footers are refused with PG_ERR_FORMAT (their bounds are
shown on the host first, by test_orc_stripes_cpu.py), and the device decodes a good section right after; TIMESTAMP
and DECIMAL(p > 18) columns are refused with PG_ERR_UNSUPPORTED."""
import pytest
import torch

import orc_stripes as S
import parquet_pages as P
from paimon_b200 import _native as N
from paimon_b200.format import read_section
from paimon_b200.types import DataField, KeyValueSchema, RowType

pytestmark = pytest.mark.gpu

PG_ERR_FORMAT = 6
CASES = S.well_formed_cases()
MALFORMED = S.malformed_cases()


def _schema(vtype):
    return KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("v", vtype, True))), ["pk"])


def _decode(files, vtype):
    readers, info = read_section(_schema(vtype), [(f.data, 0) for f in files], 1, file_format="orc")
    batches = []
    for r in readers:
        try:
            batches.append(r.read_batch())
        finally:
            r.close()
    return batches[0], info


def _check(case):
    vt = S.VTYPES[case.vtype]
    batch, info = _decode(case.files, vt.read)
    got = P.column_values(batch.value_column(1), vt.read)
    assert got == case.expected, S.first_mismatch(got, case.expected)
    assert batch.value_column(0).data[:batch.n_rows].tolist() == list(range(len(case.expected)))
    return got, info


@pytest.mark.parametrize("name", sorted(CASES))
def test_decoder_matches_the_built_stripes(name):
    case = CASES[name]()
    got, info = _check(case)
    assert info.n_chunks == case.n_tasks
    assert info.n_data_pages == case.n_streams
    if case.pyarrow:
        want = [case.arrow_view(v) for v in case.expected] if case.arrow_view else case.expected
        assert S.read_with_pyarrow(case) == want


def test_warps_decode_several_streams_of_different_codecs():
    """The many-streams section has more streams than k_orc_inflate has warps (4 CTAs of 4 warps per SM), its zstd
    chunks carry 4-stream Huffman literals, and every value comes back."""
    case = S.many_streams_case()
    warps = torch.cuda.get_device_properties(0).multi_processor_count * 16
    assert case.n_streams > warps, (case.n_streams, warps)
    assert S.zstd_literals_streams(S.compress(S.ZSTD, b"".join(S.many_streams_dictionary(0)))) == 4
    assert {S.MANY_CODECS[i % 4] for i in range(len(case.files))} == {S.ZLIB, S.ZSTD, S.LZ4, S.NONE}
    got, info = _check(case)
    assert info.n_data_pages == case.n_streams > warps


@pytest.mark.parametrize("name", sorted(MALFORMED))
def test_malformed_stream_is_a_format_error(name):
    """The section is refused with PG_ERR_FORMAT, and a good section decoded next on the same device still matches."""
    f, vtype = MALFORMED[name]()
    with pytest.raises(N.PaimonGpuError) as ei:
        _decode([f], S.VTYPES[vtype].read)
    assert ei.value.status == PG_ERR_FORMAT, str(ei.value)
    _check(S.validity_join_case())


@pytest.mark.parametrize("vt", [S.VType("TIMESTAMP(3)", S.K_TIMESTAMP, 8), S.VType("DECIMAL(18,2)", S.K_DECIMAL, 8, 20, 2)],
                         ids=["timestamp", "decimal_p20"])
def test_unmapped_orc_types_are_refused_as_unsupported(vt):
    d, vals = S.direct(list(range(10)), 7)
    sec, _ = S.short_repeat(2, 1, 10)
    f = S.kv_orc_file(vt, [S.Stripe(vals, [S.Stream(S.DATA, d), S.Stream(S.SECONDARY, sec)])])
    with pytest.raises(N.UnsupportedOnDevice):
        _decode([f], vt.read)
