"""Plain-Python restatement of the reference's field aggregators and of the two merge functions that drive them,
keyed by the LOGICAL type of a field.  TEST INFRASTRUCTURE ONLY.

This is a second yardstick next to the C oracle (oracle/paimon_oracle.c).  The oracle and the device both look at a
column through its physical type; the reference's aggregators switch on the logical type root.  Nothing here imports
oracle/ or the native library: every rule below is written from the Java sources it cites (paths under
paimon-core/src/main/java/org/apache/paimon/mergetree/compact/ unless noted).

  FieldSumAgg.java:35-163            sum, retract = subtract, negative() for a NULL accumulator
  FieldProductAgg.java:35-123        product, retract = divide
  FieldMaxAgg / FieldMinAgg          InternalRowUtils.compare (paimon-common/.../utils/InternalRowUtils.java:387-432)
  FieldLastValueAgg, FieldLastNonNullValueAgg, FieldFirstValueAgg, FieldFirstNonNullValueAgg, FieldPrimaryKeyAgg,
  FieldBoolAndAgg, FieldBoolOrAgg, FieldIgnoreRetractAgg
  FieldAggregator.java:40-54         aggReversed(acc, in) = agg(in, acc); retract() throws by default
  DecimalUtils.java:52-87, Decimal.java:182-193 (paimon-common)   DECIMAL add / subtract / fromBigDecimal
  aggregate/AggregateMergeFunction.java:80-125                     add / getResult
  PartialUpdateMergeFunction.java:121-175, 190-342                 sequence groups with aggregators
  ReducerMergeFunctionWrapper.java:45-73                           a key with one record passes through

Values: Python int for the integer types, DATE / TIME / TIMESTAMP and for DECIMAL (the unscaled value);
numpy.float32 / numpy.float64 for FLOAT / DOUBLE (one IEEE operation per step, warnings off); bytes for CHAR / VARCHAR /
BINARY / VARBINARY; bool for BOOLEAN; None for NULL.
"""
from __future__ import annotations

import struct
from fractions import Fraction
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

INSERT, UPDATE_BEFORE, UPDATE_AFTER, DELETE = 0, 1, 2, 3

_INT_BITS = {"TINYINT": 8, "SMALLINT": 16, "INT": 32, "INTEGER": 32, "BIGINT": 64,
             "DATE": 32, "TIME": 32, "TIMESTAMP": 64}
_NUMERIC = {"TINYINT", "SMALLINT", "INT", "INTEGER", "BIGINT", "FLOAT", "DOUBLE", "DECIMAL"}
_BYTES = {"CHAR", "VARCHAR", "STRING", "BINARY", "VARBINARY", "BYTES"}
_SUPPORTS_RETRACT = {"sum", "product", "last_value", "last_non_null_value", "primary-key"}

NOT_RETRACTABLE = ("Aggregate function does not support retraction, If you allow this function to ignore retraction "
                   "messages, you can configure 'fields.${field_name}.ignore-retract'='true'.")


class JavaException(Exception):
    """What the Java merge function would have thrown; str() is the exception's message."""


def type_root(logical: str) -> str:
    root = logical.upper().split("(")[0].strip()
    return "INT" if root == "INTEGER" else root


def decimal_ps(logical: str) -> Tuple[int, int]:
    """DecimalType(precision, scale); DECIMAL alone is DECIMAL(10, 0) (paimon-api/.../types/DecimalType.java:41-45)."""
    if "(" not in logical:
        return 10, 0
    args = [int(a) for a in logical[logical.index("(") + 1: logical.rindex(")")].split(",")]
    return args[0], args[1] if len(args) > 1 else 0


def wrap(v: int, bits: int) -> int:
    """The Java narrowing cast to a `bits`-wide two's complement integer."""
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def java_div(a: int, b: int) -> int:
    """Java integer division: truncates toward zero; / 0 throws."""
    if b == 0:
        raise JavaException("/ by zero")
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


# ---- DECIMAL: the unscaled value is an exact Python int

def round_half_up(f: Fraction) -> int:
    """RoundingMode.HALF_UP: ties go away from zero."""
    q = (abs(f.numerator) * 2 + f.denominator) // (2 * f.denominator)
    return -q if f < 0 else q


def _digits(v: int) -> int:                    # BigDecimal.precision() of an unscaled value (0 has one digit)
    return len(str(abs(v)))


def from_big_decimal(f: Fraction, p: int, s: int) -> Optional[int]:
    """Decimal.fromBigDecimal(bd, p, s) with bd = f: setScale(s, HALF_UP), NULL when it has more than p digits."""
    q = round_half_up(f * 10 ** s)
    return None if _digits(q) > p else q


def decimal_add(a: int, b: int, p: int, s: int) -> Optional[int]:
    """DecimalUtils.add: Math.addExact on the unscaled longs, kept whatever its digit count (fromUnscaledLong does not
    check the precision); on long overflow the BigDecimal fallback has more than 18 >= p digits -> NULL."""
    r = a + b
    return r if -(1 << 63) <= r < (1 << 63) else from_big_decimal(Fraction(r, 10 ** s), p, s)


def decimal_subtract(a: int, b: int, p: int, s: int) -> Optional[int]:
    r = a - b
    return r if -(1 << 63) <= r < (1 << 63) else from_big_decimal(Fraction(r, 10 ** s), p, s)


def decimal_multiply(a: int, b: int, p: int, s: int) -> Optional[int]:
    """BigDecimal.multiply is exact (scale 2s); fromBigDecimal rescales to s HALF_UP."""
    return from_big_decimal(Fraction(a * b, 10 ** (2 * s)), p, s)


def decimal_divide(a: int, b: int, p: int, s: int) -> Optional[int]:
    """BigDecimal.divide(BigDecimal): the exact quotient, or ArithmeticException."""
    if b == 0:
        raise JavaException("Division undefined" if a == 0 else "Division by zero")
    q = Fraction(a, b)                          # (a / 10^s) / (b / 10^s)
    d = q.denominator
    for f in (2, 5):
        while d % f == 0:
            d //= f
    if d != 1:
        raise JavaException("Non-terminating decimal expansion; no exact representable decimal result.")
    return from_big_decimal(q, p, s)


def decimal_negate(a: int, p: int, s: int) -> Optional[int]:
    return from_big_decimal(Fraction(-a, 10 ** s), p, s)


# ---- comparison (InternalRowUtils.compare)

def _float_bits(v, root: str) -> int:
    """Float.floatToIntBits / Double.doubleToLongBits: NaN canonicalised, as a signed integer."""
    if root == "FLOAT":
        if np.isnan(v):
            return 0x7fc00000
        return struct.unpack("<i", np.float32(v).tobytes())[0]
    if np.isnan(v):
        return 0x7ff8000000000000
    return struct.unpack("<q", np.float64(v).tobytes())[0]


def java_compare(root: str, a, b) -> int:
    if root in ("FLOAT", "DOUBLE"):             # Float.compare / Double.compare: -0.0 < 0.0, NaN largest
        if a < b:
            return -1
        if a > b:
            return 1
        x, y = _float_bits(a, root), _float_bits(b, root)
        return (x > y) - (x < y)
    if root in _BYTES:                          # unsigned bytes, then length
        for x, y in zip(a, b):
            if x != y:
                return -1 if x < y else 1
        return (len(a) > len(b)) - (len(a) < len(b))
    if root == "BOOLEAN":
        raise JavaException("Incomparable type: BOOLEAN")
    return (a > b) - (a < b)                    # integers, DATE / TIME / TIMESTAMP, DECIMAL at one scale


# ---- one field

class FieldAgg:
    """FieldAggregator for one field: agg / aggReversed / retract, with the per-key state of first_value."""

    def __init__(self, name: str, logical: str, ignore_retract: bool = False):
        self.name = name
        self.logical = logical
        self.root = type_root(logical)
        self.ignore_retract = ignore_retract
        self.initialized = False
        if name in ("sum", "product") and self.root not in _NUMERIC:        # FieldSumAggFactory / FieldProductAggFactory
            raise ValueError(f"Data type for {name} column must be 'NumericType' but was '{logical}'.")
        if name in ("bool_and", "bool_or") and self.root != "BOOLEAN":
            raise ValueError(f"Data type for {name.replace('_', ' ')} column must be 'BooleanType' but was "
                             f"'{logical}'.")
        if name in ("max", "min") and self.root == "BOOLEAN":
            raise ValueError("Incomparable type: BOOLEAN")

    def reset(self) -> None:
        self.initialized = False

    def _arith(self, op: str, a, b):
        root = self.root
        if root == "DECIMAL":
            p, s = decimal_ps(self.logical)
            return {"+": decimal_add, "-": decimal_subtract, "*": decimal_multiply, "/": decimal_divide}[op](a, b, p, s)
        if root in ("FLOAT", "DOUBLE"):
            t = np.float32 if root == "FLOAT" else np.float64
            x, y = t(a), t(b)
            with np.errstate(all="ignore"):
                r = {"+": np.add, "-": np.subtract, "*": np.multiply, "/": np.divide}[op](x, y)
            return t(r)
        bits = _INT_BITS[root]
        if op == "/":
            return wrap(java_div(a, b), bits)
        return wrap({"+": a + b, "-": a - b, "*": a * b}[op], bits)

    def _negative(self, v):
        if v is None:
            return None
        if self.root == "DECIMAL":
            return decimal_negate(v, *decimal_ps(self.logical))
        if self.root in ("FLOAT", "DOUBLE"):
            return np.negative(v)
        return wrap(-v, _INT_BITS[self.root])

    def agg(self, acc, inp):
        n = self.name
        if n in ("sum", "product", "max", "min", "bool_and", "bool_or"):
            if acc is None or inp is None:
                return inp if acc is None else acc
            if n == "sum":
                return self._arith("+", acc, inp)
            if n == "product":
                return self._arith("*", acc, inp)
            if n == "max":
                return inp if java_compare(self.root, acc, inp) < 0 else acc
            if n == "min":
                return acc if java_compare(self.root, acc, inp) < 0 else inp
            return (acc and inp) if n == "bool_and" else (acc or inp)
        if n in ("last_value", "primary-key"):
            return inp
        if n == "last_non_null_value":
            return acc if inp is None else inp
        if n == "first_value":
            if not self.initialized:
                self.initialized = True
                return inp
            return acc
        if n == "first_non_null_value":
            if not self.initialized and inp is not None:
                self.initialized = True
                return inp
            return acc
        raise ValueError(f"aggregate function {n} is not restated here")

    def agg_reversed(self, acc, inp):
        return self.agg(inp, acc)

    def retract(self, acc, inp):
        if self.ignore_retract:                                             # FieldIgnoreRetractAgg
            return acc
        n = self.name
        if n == "sum":
            if acc is None or inp is None:
                return self._negative(inp) if acc is None else acc
            return self._arith("-", acc, inp)
        if n == "product":
            if acc is None or inp is None:
                return acc
            return self._arith("/", acc, inp)
        if n == "last_value":
            return None
        if n == "last_non_null_value":
            return acc if inp is None else None
        if n == "primary-key":
            return inp
        raise JavaException(NOT_RETRACTABLE)


# ---- merge functions

def _agg_name(options: Dict[str, str], field: str, default: Optional[str]) -> Optional[str]:
    return (options.get(f"fields.{field}.aggregate-function") or options.get("fields.default-aggregate-function")
            or default)


def _true(options: Dict[str, str], key: str) -> bool:
    return str(options.get(key, "false")).lower() == "true"


class AggregateReference:
    """AggregateMergeFunction under ReducerMergeFunctionWrapper, for one key at a time.

    `fields` are (name, logical type) pairs of the value row; `options` are the table options the reference
    factory reads (fields.<f>.aggregate-function, fields.default-aggregate-function, fields.<f>.ignore-retract,
    aggregation.remove-record-on-delete)."""

    def __init__(self, fields: Sequence[Tuple[str, str]], primary_keys: Sequence[str], options: Dict[str, str]):
        self.fields = list(fields)
        self.remove_record_on_delete = _true(options, "aggregation.remove-record-on-delete")
        self.aggs = []
        for name, logical in self.fields:                                   # getAggFuncName :179-204
            fn = "primary-key" if name in primary_keys else _agg_name(options, name, "last_non_null_value")
            self.aggs.append(FieldAgg(fn, logical, _true(options, f"fields.{name}.ignore-retract")))

    def merge(self, records: Sequence[Tuple[int, Sequence]]) -> Tuple[int, list]:
        """records: (row kind, value row) of one key in sequence order -> (row kind, value row) of the result."""
        if len(records) == 1:                                               # ReducerMergeFunctionWrapper
            return records[0][0], list(records[0][1])
        for a in self.aggs:
            a.reset()
        row = [None] * len(self.fields)
        delete_row = False
        for kind, value in records:                                         # AggregateMergeFunction.add :80-101
            delete_row = self.remove_record_on_delete and kind == DELETE
            if delete_row:
                row = list(value)
                continue
            retract = kind in (UPDATE_BEFORE, DELETE)
            row = [a.retract(acc, v) if retract else a.agg(acc, v) for a, acc, v in zip(self.aggs, row, value)]
        return (DELETE if delete_row else INSERT), row


class PartialUpdateReference:
    """PartialUpdateMergeFunction with sequence groups ('fields.<seq>.sequence-group' = '<f>,...') whose fields may
    have aggregate functions, under ReducerMergeFunctionWrapper.  Sequence fields are compared NULL-first."""

    def __init__(self, fields: Sequence[Tuple[str, str]], primary_keys: Sequence[str], options: Dict[str, str]):
        self.fields = list(fields)
        names = [f[0] for f in self.fields]
        self.group_of: List[Optional[List[int]]] = [None] * len(names)    # per field: sequence fields of its group
        self.seq_fields = set()
        for k, v in options.items():
            if k.startswith("fields.") and k.endswith(".sequence-group"):
                seq = [names.index(n.strip()) for n in k[len("fields."):-len(".sequence-group")].split(",")]
                for f in [names.index(n.strip()) for n in v.split(",")] + seq:
                    self.group_of[f] = seq
                self.seq_fields.update(seq)
        self.aggs: List[Optional[FieldAgg]] = []
        for i, (name, logical) in enumerate(self.fields):
            if i in self.seq_fields:
                fn = None
            elif name in primary_keys:
                fn = "primary-key"
            else:
                fn = _agg_name(options, name, None)
            self.aggs.append(None if fn is None else FieldAgg(fn, logical, _true(options, f"fields.{name}.ignore-retract")))

    @staticmethod
    def _compare(value, row, seq) -> int:
        for f in seq:
            a, b = value[f], row[f]
            if a is None or b is None:
                if (a is None) != (b is None):
                    return -1 if a is None else 1
                continue
            if a != b:
                return -1 if a < b else 1
        return 0

    def merge(self, records: Sequence[Tuple[int, Sequence]]) -> Tuple[int, list]:
        if len(records) == 1:
            return records[0][0], list(records[0][1])
        for a in self.aggs:
            if a is not None:
                a.reset()
        row = [None] * len(self.fields)
        meet_insert = filled = False
        for kind, value in records:
            if kind in (UPDATE_BEFORE, DELETE):                             # add :124-144 -> retractWithSequenceGroup
                if not filled:
                    row = list(value)
                    filled = True
                empty, updated = set(), set()
                for i in range(len(row)):
                    seq = self.group_of[i]
                    if seq is None or self._empty(value, seq, empty):
                        continue
                    if self._compare(value, row, seq) >= 0:
                        if i in seq:
                            for f in seq:
                                if f not in updated:
                                    row[f] = value[f]
                                    updated.add(f)
                        else:
                            row[i] = None if self.aggs[i] is None else self.aggs[i].retract(row[i], value[i])
                    elif self.aggs[i] is not None:
                        row[i] = self.aggs[i].retract(row[i], value[i])
                continue
            empty = set()                                                   # updateWithSequenceGroup :190-247
            for i in range(len(row)):
                seq, a, v = self.group_of[i], self.aggs[i], value[i]
                if seq is None:
                    if a is not None:
                        row[i] = a.agg(row[i], v)
                    elif v is not None:
                        row[i] = v
                    continue
                if self._empty(value, seq, empty):
                    continue
                if self._compare(value, row, seq) >= 0:
                    if i in seq:
                        for f in seq:
                            row[f] = value[f]
                        continue
                    row[i] = v if a is None else a.agg(row[i], v)
                elif a is not None:
                    row[i] = a.agg_reversed(row[i], v)
            meet_insert = filled = True
        return (INSERT if meet_insert else DELETE), row

    @staticmethod
    def _empty(value, seq, empty) -> bool:                                  # isEmptySequenceGroup :249-269
        if seq[0] in empty:
            return True
        if any(value[f] is not None for f in seq):
            return False
        empty.update(seq)
        return True
