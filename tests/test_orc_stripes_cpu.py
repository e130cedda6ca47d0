"""The host build of the ORC decode path (orc_meta.cc + the chunk decoders + orc_device.cuh, the sources the device
compiles) on hand-built stripes (orc_stripes.py): every RLE v2 sub-encoding at its header-field edges, RLE v1 runs,
literals and 10-byte varints, byte RLE and boolean streams, DECIMAL per-value scales, DIRECT and DICTIONARY strings,
floats by bit pattern, compression chunks mixed original / compressed and cut mid-value under ZLIB, ZSTD and LZ4.  Each
case must equal the builder's values and pyarrow.orc's reading of the same bytes.  Malformed streams and footers —
truncated streams, dictionary ids and lengths out of range, bad patch lists, broken chunks, DECIMAL scales out of range
and dictionary sizes beyond the stripe's rows — must be refused, and in bounded time (a wrong bound here would hang one
device thread)."""
import pytest

import orc_stripes as S
import orc_util

CASES = S.well_formed_cases()
MALFORMED = S.malformed_cases()


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return orc_util.build(str(tmp_path_factory.mktemp("orc_stripes")))


def _decode(lib, f: S.OrcFile, vtype: str):
    vt = S.VTYPES[vtype]
    n, cols = orc_util.decode(lib, f.data, [8, 8, 1, 8, vt.width])
    assert n == len(f.expected)
    return cols, S.host_values(cols[4], vt, n)


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_decoder_matches_the_built_stripes(lib, name):
    case = CASES[name]()
    got, key0 = [], 0
    for f in case.files:
        cols, vals = _decode(lib, f, case.vtype)
        assert cols[3][0].tolist() == list(range(key0, key0 + len(vals)))
        assert cols[1][1].all() and cols[3][1].all()
        got += vals
        key0 += len(vals)
    assert got == case.expected, S.first_mismatch(got, case.expected)
    if case.pyarrow:
        arrow = S.read_with_pyarrow(case)
        want = [case.arrow_view(v) for v in case.expected] if case.arrow_view else case.expected
        assert arrow == want, "pyarrow: " + S.first_mismatch(arrow, want)


@pytest.mark.parametrize("name", sorted(MALFORMED))
def test_malformed_stream_is_refused(lib, name):
    f, vtype = MALFORMED[name]()
    with pytest.raises(RuntimeError):
        _decode(lib, f, vtype)


def test_builder_runs_match_the_specification_examples():
    """The RLE v2 encoders reproduce the worked examples of the ORC specification byte for byte, so the builder is
    pinned to the format rather than to the decoder it judges."""
    assert S.short_repeat(10000, 2, 5, signed=False)[0] == bytes([0x0A, 0x27, 0x10])
    assert S.direct([23713, 43806, 57005, 48879], S.width_code(16), signed=False)[0] == \
        bytes([0x5E, 0x03, 0x5C, 0xA1, 0xAB, 0x1E, 0xDE, 0xAD, 0xBE, 0xEF])
    b, vals = S.delta(2, 1, [2, 2, 4, 2, 4, 2, 4, 6], S.width_code(4), signed=False)
    assert vals == [2, 3, 5, 7, 11, 13, 17, 19, 23, 29]
    assert b == bytes([0xC6, 0x09, 0x02, 0x02, 0x22, 0x42, 0x42, 0x46])
    vals = [2030, 2000, 2020, 1000000] + list(range(2040, 2200, 10))
    b, _ = S.patched_base(vals, 2, 8, 12, 2)
    assert b == bytes([0x8E, 0x13, 0x2B, 0x21, 0x07, 0xD0, 0x1E, 0x00, 0x14, 0x70, 0x28, 0x32, 0x3C, 0x46, 0x50,
                       0x5A, 0x64, 0x6E, 0x78, 0x82, 0x8C, 0x96, 0xA0, 0xAA, 0xB4, 0xBE, 0xFC, 0xE8])
