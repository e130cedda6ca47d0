"""The device Parquet decoder on hand-built pages (parquet_pages.py), compared with the builder's expected values:
floats by bit pattern, strings by bytes, validity bit for bit, and with pyarrow's reading of the same files.  The cases
cover dictionary ids at widths 0 to 32 in RLE, bit-packed and alternating streams with 1- to 3-byte run headers through
every fixed type, STRING / BINARY and the INT -> BIGINT / FLOAT -> DOUBLE casts; RLE booleans; definition levels of
every run shape in V1 and V2 pages and pages of 1 to 63 rows whose starts fall on every bit of a validity word;
DELTA_BINARY_PACKED block shapes, miniblock widths and totals; CRCs, page statistics, unknown header fields, index pages
and V2 pages stored uncompressed under a codec.  Malformed streams (short or truncated ids, booleans and definition
levels, a dictionary page that claims more entries than it holds) are refused with PG_ERR_FORMAT."""
import io

import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_pages as P
from paimon_b200 import _native as N
from paimon_b200.format import read_section
from paimon_b200.types import DataField, KeyValueSchema, RowType

pytestmark = pytest.mark.gpu

PG_ERR_FORMAT = 6
CASES = P.well_formed_cases()
MALFORMED = P.malformed_cases()


def _schema(vtype):
    return KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("v", vtype, True))), ["pk"])


def _decode(files, vtype):
    readers, info = read_section(_schema(vtype), [(f, 0) for f in files], 1)
    batches = []
    for r in readers:
        try:
            batches.append(r.read_batch())
        finally:
            r.close()
    return batches[0], info


def _check(case):
    batch, info = _decode(case.files, case.vtype)
    got = P.column_values(batch.value_column(1), case.vtype)
    assert got == case.expected, P.first_mismatch(got, case.expected)
    assert batch.value_column(0).data[:batch.n_rows].tolist() == list(range(len(case.expected)))
    return got, info


@pytest.mark.parametrize("name", sorted(CASES))
def test_decoder_matches_the_built_pages(name):
    case = CASES[name]()
    got, info = _check(case)
    assert info.n_data_pages == case.data_pages
    assert info.n_dictionary_pages == (case.dict_pages or 0)
    if "->" in name:
        return                                         # (pyarrow reads the file type, not the widened one)
    tables = [pq.read_table(io.BytesIO(f), page_checksum_verification=case.crc) for f in case.files]
    assert got == P.arrow_values(pa.concat_tables(tables).column("v"), case.vtype)


@pytest.mark.parametrize("name", sorted(MALFORMED))
def test_malformed_stream_is_a_format_error(name):
    """The section is refused with PG_ERR_FORMAT, and a good section decoded next on the same device still matches."""
    data, vtype = MALFORMED[name]()
    with pytest.raises(N.PaimonGpuError) as ei:
        _decode([data], vtype)
    assert ei.value.status == PG_ERR_FORMAT
    _check(P.small_pages_case())
