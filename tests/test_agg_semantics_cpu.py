"""The aggregate functions against an independent reference (tests/agg_reference.py) for each LOGICAL type, on the
CPU: the reference against the reference's own known answers, the C oracle against the reference on edge-value
folds, and the factories' type checks.  The device side of the same comparison is test_gpu_aggregate_semantics.py."""
import random
import struct
import zlib

import numpy as np
import pytest

import agg_reference as R
from oracle import pyoracle
from paimon_b200.columnar import Column, KeyValueBatch, unpack_validity
from paimon_b200.merge_function import AggregateMergeFunction, PartialUpdateMergeFunction
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType, is_varlen, physical_type

F32 = lambda bits: np.frombuffer(struct.pack("<I", bits), np.float32)[0]      # noqa: E731
F64 = lambda bits: np.frombuffer(struct.pack("<Q", bits), np.float64)[0]      # noqa: E731

# ---------------------------------------------------------------------------------------------- edge values

def _ints(bits):
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    return [lo, hi, -1, 0, 1, 2, -2, lo + 1, hi - 1, 3, -3, 1 << (bits - 2), -(1 << (bits - 2))]


_FLOAT_EDGES = [0.0, F32(0x80000000), np.float32(np.inf), np.float32(-np.inf), F32(0x7fc00000), F32(0x7fc00123),
                F32(0xffc00000), F32(0x00000001), F32(0x80000001), F32(0x7f7fffff), F32(0xff7fffff), 1.0, -1.0,
                1.5, -1.5, 3.0, 1e-30, 16777216.0, 0.1]
_DOUBLE_EDGES = [0.0, F64(0x8000000000000000), np.inf, -np.inf, F64(0x7ff8000000000000), F64(0x7ff8000000000123),
                 F64(0xfff8000000000000), F64(0x0000000000000001), F64(0x8000000000000001), F64(0x7fefffffffffffff),
                 F64(0xffefffffffffffff), 1.0, -1.0, 1.5, -1.5, 3.0, 1e-300, 9007199254740992.0, 0.1]
_BYTES_EDGES = [b"", b"a", b"ab", b"b", b"\x7f", b"\x80", b"\xff", b"\xff\x00", b"\xff\xff", b"a\x00", b"\x00",
                b"\xc3\xa9", b"zz"]


def decimal_edges(p, s):
    m = 10 ** p - 1
    one = 10 ** s
    half = 5 * 10 ** (s - 1) if s else 1
    return [m, -m, 0, 1, -1, one, -one, 2 * one, -2 * one, half, -half, 3 * half, -3 * half, one + half, 10 ** (p - 1),
            -(10 ** (p - 1)), 4 * one, 8 * one, 3 * one, m // 3]


def edge_values(logical):
    root = R.type_root(logical)
    if root in R._INT_BITS:
        return _ints(R._INT_BITS[root])
    if root == "FLOAT":
        return [np.float32(v) for v in _FLOAT_EDGES]
    if root == "DOUBLE":
        return [np.float64(v) for v in _DOUBLE_EDGES]
    if root == "DECIMAL":
        return decimal_edges(*R.decimal_ps(logical))
    if root in R._BYTES:
        return list(_BYTES_EDGES)
    raise ValueError(logical)


# every aggregator a type admits (FieldAggregatorFactory + the factories' type checks)
_SELECT = ["max", "min", "first_value", "first_non_null_value", "last_value", "last_non_null_value"]
AGGS_OF = {
    "TINYINT": ["sum", "product"] + _SELECT, "SMALLINT": ["sum", "product"] + _SELECT,
    "INT": ["sum", "product"] + _SELECT, "BIGINT": ["sum", "product"] + _SELECT,
    "FLOAT": ["sum", "product"] + _SELECT, "DOUBLE": ["sum", "product"] + _SELECT,
    "DECIMAL(9,2)": ["sum", "product"] + _SELECT, "DECIMAL(18,4)": ["sum", "product"] + _SELECT,
    "DECIMAL(10,0)": ["sum", "product"] + _SELECT, "DECIMAL(15,2)": ["sum", "product"] + _SELECT,
    "DATE": _SELECT, "TIMESTAMP": _SELECT, "STRING": _SELECT, "BINARY(8)": _SELECT,
}


# ---------------------------------------------------------------------------------------------- fold generator

class Fold:
    """One table of random keys for one (type, aggregator, ignore-retract) case: the runs to merge and, per key, the
    reference's (kind, value) result."""

    def __init__(self, logical, agg, ignore_retract, n_keys, max_records, n_runs, seed, retracts=True,
                 remove_on_delete=False):
        self.logical, self.agg = logical, agg
        rng = random.Random(seed)
        vt = RowType((DataField("k", "INT", False), DataField("v", logical, True)))
        self.schema = KeyValueSchema.of(vt, ["k"])
        opts = {"fields.v.aggregate-function": agg}
        if ignore_retract:
            opts["fields.v.ignore-retract"] = "true"
        if remove_on_delete:
            opts["aggregation.remove-record-on-delete"] = "true"
        self.spec = AggregateMergeFunction.factory(opts, vt, ["k"]).create()
        ref = R.AggregateReference([("k", "INT"), ("v", logical)], ["k"], opts)
        edges = edge_values(logical)
        big = 10 ** R.decimal_ps(logical)[0] - 1 if R.type_root(logical) == "DECIMAL" else None
        rows_of_run = [[] for _ in range(n_runs)]
        self.expected = {}
        for key in range(n_keys):
            n = rng.randint(1, min(max_records, n_runs))
            kinds = [rng.choice([R.INSERT, R.INSERT, R.UPDATE_AFTER, R.UPDATE_BEFORE, R.DELETE]) if retracts
                     else R.INSERT for _ in range(n)]
            vals = [None if rng.random() < 0.1 else rng.choice(edges) for _ in range(n)]
            if big is not None and rng.random() < 0.15:
                # the largest value over and over: DECIMAL(18, s) sums cross int64 (NULL), then restart
                vals = [rng.choice([big, big, big, -big, None]) for _ in range(n)]
            records = list(zip(kinds, [(key, v) for v in vals]))
            try:
                res = ref.merge(records)
            except R.JavaException:
                records = [(R.INSERT, r) for _, r in records]            # what the reference would throw on
                res = ref.merge(records)
            self.expected[key] = res
            runs = sorted(rng.sample(range(n_runs), n))
            for j, (r, (kind, row)) in enumerate(zip(runs, records)):
                rows_of_run[r].append((key, j, kind, key, row[1]))
        self.runs = [KeyValueBatch.from_rows(self.schema, rows) for rows in rows_of_run if rows]


def cell(col: Column, i: int):
    """A cell as comparable bits: None, int, raw float bits, or bytes."""
    if not unpack_validity(col.valid, len(col))[i]:
        return None
    if is_varlen(col.type):
        return bytes(col.data[col.offsets[i]:col.offsets[i + 1]].tobytes())
    if col.type == PhysicalType.FLOAT:
        return ("f32", int(np.asarray(col.data[i:i + 1], np.float32).view(np.uint32)[0]))
    if col.type == PhysicalType.DOUBLE:
        return ("f64", int(np.asarray(col.data[i:i + 1], np.float64).view(np.uint64)[0]))
    return int(col.data[i])


def ref_cell(logical, v):
    if v is None:
        return None
    root = R.type_root(logical)
    if root == "FLOAT":
        return ("f32", int(np.float32(v).view(np.uint32)))
    if root == "DOUBLE":
        return ("f64", int(np.float64(v).view(np.uint64)))
    return v


def is_nan_bits(c):
    if not isinstance(c, tuple):
        return False
    return np.isnan(F32(c[1]) if c[0] == "f32" else F64(c[1]))


def same_value(agg, got, want):
    """Arithmetic results (sum / product) bit for bit except that all NaNs are equal (neither Java nor the H100 fix
    the payload of a NaN an add or multiply returns); selected inputs bit for bit, NaN payload included."""
    if agg in ("sum", "product") and is_nan_bits(got) and is_nan_bits(want):
        return True
    return got == want


def check_against_reference(fold: Fold, batch: KeyValueBatch):
    """Key set, row kinds and the folded value column of `batch` against the reference."""
    keys = [int(k) for k in batch.key_column(0).data[: batch.n_rows]]
    assert keys == sorted(fold.expected), "key set differs"
    kinds = batch.value_kinds
    vcol = batch.value_column(1)
    bad = []
    for i, k in enumerate(keys):
        want_kind, want_row = fold.expected[k]
        got = cell(vcol, i)
        want = ref_cell(fold.logical, want_row[1])
        if int(kinds[i]) != want_kind or not same_value(fold.agg, got, want):
            bad.append((k, int(kinds[i]), got, want_kind, want))
    assert not bad, f"{len(bad)} keys differ, first: {bad[:3]}"


# ---------------------------------------------------------------------------------------------- known answers

# FieldAggregatorTest.java:415-561: (logical type, aggregator, op, accumulator, input, expected); DECIMAL is
# DECIMAL(10, 0), whose unscaled value is the number itself (FieldAggregatorTest.toDecimal :563-566)
KNOWN = []
for _t in ["TINYINT", "SMALLINT", "INT", "BIGINT", "FLOAT", "DOUBLE", "DECIMAL"]:
    KNOWN += [(_t, "sum", "agg", None, 10, 10), (_t, "sum", "agg", 1, 10, 11),
              (_t, "sum", "retract", 10, 5, 5), (_t, "sum", "retract", None, 5, -5),
              (_t, "product", "agg", None, 10, 10), (_t, "product", "agg", 1, 10, 10),
              (_t, "product", "retract", 10, 5, 2), (_t, "product", "retract", None, 5, None)]
KNOWN += [("INT", "max", "agg", 1, 10, 10), ("INT", "min", "agg", 1, 10, 1)]

# hand-worked DECIMAL(15,2) cases: unscaled values, scale 2
DEC15 = "DECIMAL(15,2)"
HAND_WORKED = [
    ("product", "agg", 150, 200, 300),                           # 1.50 * 2.00 = 3.00
    ("product", "agg", 105, 50, 53),                             # 0.525 -> 0.53 (HALF_UP tie)
    ("product", "agg", -105, 50, -53),                           # -0.525 -> -0.53 (away from zero)
    ("product", "agg", 15, 5, 1),                                # 0.0075 -> 0.01
    ("product", "agg", 999_999_999_999_999, 1000, None),         # 99999999999999.90: 16 digits > 15 -> NULL
    ("product", "agg", 99_999_999_999_999, 100, 99_999_999_999_999),   # 999999999999.99 * 1.00: fits
    ("sum", "agg", 9_223_372_036_854_775_000, 900, None),        # crosses int64 -> NULL
    ("sum", "agg", 999_999_999_999_999, 999_999_999_999_999, 1_999_999_999_999_998),   # over p digits: kept
    ("sum", "retract", -9_223_372_036_854_775_000, 900, None),   # subtract crosses int64 -> NULL
    ("sum", "retract", None, 999_999_999_999_999, -999_999_999_999_999),
    ("product", "retract", 1000, 400, 250),                      # 10.00 / 4.00 = 2.50
    ("product", "retract", 100, 800, 13),                        # 1.00 / 8.00 = 0.125 -> 0.13
    ("product", "retract", -100, 800, -13),                      # -0.125 -> -0.13
    ("product", "retract", 999_999_999_999_999, 1, None),        # / 0.01: 17 digits -> NULL
]
HAND_WORKED_ERRORS = [
    (100, 300, "Non-terminating decimal expansion; no exact representable decimal result."),   # 1.00 / 3.00
    (100, 0, "Division by zero"),
    (0, 0, "Division undefined"),
]


def _python(logical, v):
    root = R.type_root(logical)
    if v is None:
        return None
    return np.float32(v) if root == "FLOAT" else np.float64(v) if root == "DOUBLE" else v


def _oracle_two_records(logical, agg, op, acc, inp):
    """agg(acc, inp) / retract(acc, inp) through the oracle: one key, an INSERT of acc and then inp."""
    vt = RowType((DataField("k", "INT", False), DataField("v", logical, True)))
    schema = KeyValueSchema.of(vt, ["k"])
    spec = AggregateMergeFunction.factory({"fields.v.aggregate-function": agg}, vt, ["k"]).create()
    kind = R.INSERT if op == "agg" else R.UPDATE_BEFORE
    runs = [KeyValueBatch.from_rows(schema, [(1, 0, R.INSERT, 1, acc)]),
            KeyValueBatch.from_rows(schema, [(1, 1, kind, 1, inp)])]
    out = pyoracle.merge(schema, spec, runs)
    return cell(out.value_column(1), 0)


@pytest.mark.parametrize("logical,agg,op,acc,inp,want", KNOWN)
def test_known_answers(logical, agg, op, acc, inp, want):
    a = R.FieldAgg(agg, logical)
    fn = a.agg if op == "agg" else a.retract
    got = fn(_python(logical, acc), _python(logical, inp))
    assert ref_cell(logical, got) == ref_cell(logical, _python(logical, want))
    assert _oracle_two_records(logical, agg, op, acc, inp) == ref_cell(logical, _python(logical, want))


@pytest.mark.parametrize("agg,op,acc,inp,want", HAND_WORKED)
def test_decimal_hand_worked(agg, op, acc, inp, want):
    a = R.FieldAgg(agg, DEC15)
    assert (a.agg if op == "agg" else a.retract)(acc, inp) == want
    assert _oracle_two_records(DEC15, agg, op, acc, inp) == want


def test_decimal_sum_restarts_after_null():
    """After an overflow to NULL the next agg starts from its input (accumulator == null ? inputField)."""
    a = R.FieldAgg("sum", DEC15)
    acc = a.agg(9_223_372_036_854_775_000, 900)
    assert acc is None and a.agg(acc, 5) == 5
    vt = RowType((DataField("k", "INT", False), DataField("v", DEC15, True)))
    schema = KeyValueSchema.of(vt, ["k"])
    spec = AggregateMergeFunction.factory({"fields.v.aggregate-function": "sum"}, vt, ["k"]).create()
    runs = [KeyValueBatch.from_rows(schema, [(1, j, R.INSERT, 1, v)])
            for j, v in enumerate([9_223_372_036_854_775_000, 900, 5, 7])]
    assert pyoracle.merge(schema, spec, runs).to_rows() == [(1, 3, R.INSERT, 1, 12)]


@pytest.mark.parametrize("acc,inp,msg", HAND_WORKED_ERRORS)
def test_decimal_retract_divide_errors(acc, inp, msg):
    with pytest.raises(R.JavaException, match=msg[:20]):
        R.FieldAgg("product", DEC15).retract(acc, inp)
    with pytest.raises(pyoracle.OracleError, match=msg[:20]):
        _oracle_two_records(DEC15, "product", "retract", acc, inp)


def test_integer_edges():
    """Java wrap-around for every width, MIN / -1 and / 0 in the product retract."""
    for t, bits in [("TINYINT", 8), ("SMALLINT", 16), ("INT", 32), ("BIGINT", 64)]:
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
        assert R.FieldAgg("sum", t).agg(hi, 1) == lo
        assert R.FieldAgg("product", t).agg(hi, 2) == -2
        assert R.FieldAgg("product", t).retract(lo, -1) == lo
        assert R.FieldAgg("product", t).retract(-7, 2) == -3
        assert R.FieldAgg("sum", t).retract(None, lo) == lo
        with pytest.raises(R.JavaException, match="/ by zero"):
            R.FieldAgg("product", t).retract(5, 0)


def test_float_order():
    """Float.compare: -0.0 < 0.0 and NaN above +inf; max / min return the chosen input verbatim."""
    nan1, nan2 = F32(0x7fc00123), F32(0x7fc00456)
    mx, mn = R.FieldAgg("max", "FLOAT"), R.FieldAgg("min", "FLOAT")
    assert ref_cell("FLOAT", mx.agg(np.float32(0.0), F32(0x80000000))) == ("f32", 0)
    assert ref_cell("FLOAT", mn.agg(np.float32(0.0), F32(0x80000000))) == ("f32", 0x80000000)
    assert ref_cell("FLOAT", mx.agg(nan1, nan2)) == ("f32", 0x7fc00123)       # equal: the accumulator stays
    assert ref_cell("FLOAT", mn.agg(nan1, nan2)) == ("f32", 0x7fc00456)       # equal: the input wins
    assert ref_cell("FLOAT", mx.agg(np.float32(np.inf), nan1)) == ("f32", 0x7fc00123)


# ---------------------------------------------------------------------------------------------- oracle vs reference

CASES = [(t, a) for t, aggs in AGGS_OF.items() for a in aggs]


@pytest.mark.parametrize("logical,agg", CASES)
@pytest.mark.parametrize("mode", ["insert_only", "retract", "ignore_retract"])
def test_oracle_matches_reference(logical, agg, mode):
    fold = Fold(logical, agg, mode == "ignore_retract", n_keys=300, max_records=12, n_runs=12,
                seed=zlib.crc32(f"{logical}/{agg}/{mode}".encode()), retracts=mode != "insert_only")
    check_against_reference(fold, pyoracle.merge(fold.schema, fold.spec, fold.runs))


@pytest.mark.parametrize("logical", ["DECIMAL(18,4)", "FLOAT", "INT"])
def test_oracle_remove_record_on_delete(logical):
    fold = Fold(logical, "sum", False, n_keys=300, max_records=8, n_runs=8, seed=7, remove_on_delete=True)
    check_against_reference(fold, pyoracle.merge(fold.schema, fold.spec, fold.runs))


# ---------------------------------------------------------------------------------------------- factory validation

@pytest.mark.parametrize("logical", ["DATE", "TIME", "TIMESTAMP", "TIMESTAMP(3)"])
@pytest.mark.parametrize("agg", ["sum", "product"])
def test_sum_product_need_numeric(logical, agg):
    vt = RowType((DataField("k", "INT", False), DataField("v", logical, True)))
    msg = f"Data type for {agg} column must be 'NumericType'"
    with pytest.raises(ValueError, match=msg):
        R.FieldAgg(agg, logical)
    with pytest.raises(ValueError, match=msg):
        AggregateMergeFunction.factory({"fields.v.aggregate-function": agg}, vt, ["k"]).create()
    vt3 = RowType((DataField("k", "INT", False), DataField("g", "BIGINT", True), DataField("v", logical, True)))
    with pytest.raises(ValueError, match=msg):
        PartialUpdateMergeFunction.factory({"fields.g.sequence-group": "v", "fields.v.aggregate-function": agg},
                                           vt3, ["k"]).create()


@pytest.mark.parametrize("logical", ["DATE", "TIMESTAMP", "DECIMAL(9,2)", "STRING"])
def test_max_min_accepted(logical):
    vt = RowType((DataField("k", "INT", False), DataField("v", logical, True)))
    for agg in ("max", "min"):
        AggregateMergeFunction.factory({"fields.v.aggregate-function": agg}, vt, ["k"]).create()
        R.FieldAgg(agg, logical)


@pytest.mark.parametrize("logical", ["DECIMAL(38,2)", "DECIMAL(19,0)", "TIMESTAMP(9)", "TIMESTAMP(7)"])
def test_physical_type_refuses_wide_types(logical):
    with pytest.raises(ValueError, match="unsupported type"):
        physical_type(logical)


def test_decimal_descriptor_in_spec():
    vt = RowType((DataField("k", "INT", False), DataField("a", "DECIMAL(15,2)", True), DataField("b", "BIGINT", True),
                  DataField("c", "DECIMAL", True)))
    spec = AggregateMergeFunction.factory({"fields.a.aggregate-function": "sum"}, vt, ["k"]).create()
    assert spec.decimal == [0, 15 << 8 | 2, 0, 10 << 8]
    assert physical_type("DECIMAL(18,4)") == PhysicalType.INT64 and physical_type("TIMESTAMP(6)") == PhysicalType.INT64
    vt2 = RowType((DataField("k", "INT", False), DataField("b", "BIGINT", True)))
    assert AggregateMergeFunction.factory({}, vt2, ["k"]).create().decimal == []
