"""The hand-built Parquet pages of parquet_pages.py, read by pyarrow: every well-formed case must decode to the
builder's expected values (with CRC verification where the pages carry CRCs).  This checks the builder itself, so the
device tests that use it compare the decoder with a reference that a second reader agrees with."""
import io

import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_pages as P

CASES = P.well_formed_cases()


def _read(case):
    tables = [pq.read_table(io.BytesIO(f), page_checksum_verification=case.crc) for f in case.files]
    return pa.concat_tables(tables)


@pytest.mark.parametrize("name", sorted(CASES))
def test_pyarrow_reads_the_builders_values(name):
    case = CASES[name]()
    assert case.pyarrow, "every well-formed case here is one pyarrow reads"
    t = _read(case)
    got = P.arrow_values(t.column("v"), case.vtype if name not in ("dict_INT->BIGINT", "dict_FLOAT->DOUBLE") else
                         {"dict_INT->BIGINT": "INT", "dict_FLOAT->DOUBLE": "FLOAT"}[name])
    want = case.expected
    if name == "dict_FLOAT->DOUBLE":                   # pyarrow reads the file type: widen its bit patterns the same way
        got = [None if g is None else b for g, b in zip(got, P._f32_to_f64_bits([g or 0 for g in got]))]
    assert got == want, P.first_mismatch(got, want)
    keys = t.column("pk").to_pylist()
    assert keys == list(range(len(want)))
    assert t.column("_SEQUENCE_NUMBER").to_pylist() == [k - k0 for f, k0 in _file_starts(case) for k in range(k0, k0 + f)]


def _file_starts(case):
    out, k0 = [], 0
    for f in case.files:
        n = pq.ParquetFile(io.BytesIO(f)).metadata.num_rows
        out.append((n, k0))
        k0 += n
    return out


def test_crc_is_checked_by_pyarrow():
    """A flipped byte in a page body that carries a CRC is refused by pyarrow: the builder's CRCs are real."""
    case = P.headers_case(P.UNCOMPRESSED)
    blob = bytearray(case.files[0])
    value = next(v for v in case.expected if v is not None and len(v) >= 4)
    at = bytes(blob).rfind(value)                      # a value of the last page that holds it: flip one of its bits
    assert at > 0
    blob[at] ^= 1
    with pytest.raises(OSError):
        pq.read_table(io.BytesIO(bytes(blob)), page_checksum_verification=True)


def test_thrift_writer_field_headers():
    w = P.ThriftWriter()
    w.i32(1, -1)
    w.i32(16, 3)              # delta 15: still short form
    w.i32(40, 0)              # delta 24: long form
    w.i32(41, 1, long_form=True)
    assert w.stop() == bytes([0x15, 0x01, 0xF5, 0x06, 0x05, 0x50, 0x00, 0x05, 0x52, 0x02, 0x00])


def test_hybrid_and_delta_encoders_on_spec_examples():
    # Encodings.md: the bit-packed example, values 0..7 at width 3
    assert P.hybrid(3, [("packed", list(range(8)))]) == bytes([0x03, 0x88, 0xC6, 0xFA])
    assert P.hybrid(3, [("rle", 300, 5)]) == bytes([0xD8, 0x04, 0x05])
    # Encodings.md DELTA_BINARY_PACKED example 1: 1..5 -> header, min delta 1, widths 0
    assert P.delta_binary_packed([1, 2, 3, 4, 5], 32) == bytes([0x80, 0x01, 0x04, 0x05, 0x02, 0x02, 0, 0, 0, 0])


@pytest.mark.parametrize("name", sorted(P.malformed_cases()))
def test_pyarrow_refuses_the_malformed_streams(name):
    """The malformed files the device decoder must refuse are refused by pyarrow too: they are malformed, not merely
    unusual."""
    data, _ = P.malformed_cases()[name]()
    with pytest.raises((OSError, pa.ArrowInvalid)):
        pq.read_table(io.BytesIO(data))
