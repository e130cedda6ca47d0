"""Type vocabulary of the hot path.

Mirrors the parts of the reference's type system that decide the physical layout of a
``KeyValue`` data file (reference: paimon-api/src/main/java/org/apache/paimon/types/RowKind.java:35-56,
paimon-core/src/main/java/org/apache/paimon/KeyValue.java:130-138,
paimon-api/src/main/java/org/apache/paimon/table/SpecialFields.java:74-86,
paimon-format/src/main/java/org/apache/paimon/format/parquet/ParquetSchemaConverter.java:76-160).
"""
from __future__ import annotations

import enum
from dataclasses import dataclass, field
from typing import List, Sequence

import numpy as np


class RowKind(enum.IntEnum):
    """RowKind byte values (RowKind.java:35-56)."""

    INSERT = 0
    UPDATE_BEFORE = 1
    UPDATE_AFTER = 2
    DELETE = 3

    def is_retract(self) -> bool:  # RowKind.java:101-103
        return self in (RowKind.UPDATE_BEFORE, RowKind.DELETE)

    def is_add(self) -> bool:  # RowKind.java:105-108
        return self in (RowKind.INSERT, RowKind.UPDATE_AFTER)


class PhysicalType(enum.IntEnum):
    """Physical column types understood by the C ABI (include/paimon_gpu.h ``pg_type``)."""

    INT8 = 1
    INT16 = 2
    INT32 = 3
    INT64 = 4
    FLOAT = 5
    DOUBLE = 6
    BOOL = 7      # one byte per value (HeapBooleanVector layout)
    STRING = 8    # int32 offsets + bytes (CHAR / VARCHAR)
    BINARY = 9    # int32 offsets + bytes (BINARY / VARBINARY)


_NP = {
    PhysicalType.INT8: np.int8, PhysicalType.INT16: np.int16, PhysicalType.INT32: np.int32,
    PhysicalType.INT64: np.int64, PhysicalType.FLOAT: np.float32, PhysicalType.DOUBLE: np.float64,
    PhysicalType.BOOL: np.uint8, PhysicalType.STRING: np.uint8, PhysicalType.BINARY: np.uint8,
}

# Paimon logical type root -> physical type.  DATE / TIME are INT32, TIMESTAMP(p<=6) and
# DECIMAL(p<=18) are INT64 (unscaled), exactly as the reference's Parquet mapping stores them.
_LOGICAL = {
    "TINYINT": PhysicalType.INT8, "SMALLINT": PhysicalType.INT16, "INT": PhysicalType.INT32,
    "INTEGER": PhysicalType.INT32, "DATE": PhysicalType.INT32, "TIME": PhysicalType.INT32,
    "BIGINT": PhysicalType.INT64, "TIMESTAMP": PhysicalType.INT64, "DECIMAL": PhysicalType.INT64,
    "FLOAT": PhysicalType.FLOAT, "DOUBLE": PhysicalType.DOUBLE, "BOOLEAN": PhysicalType.BOOL,
    "STRING": PhysicalType.STRING, "VARCHAR": PhysicalType.STRING, "CHAR": PhysicalType.STRING,
    "BINARY": PhysicalType.BINARY, "VARBINARY": PhysicalType.BINARY, "BYTES": PhysicalType.BINARY,
}


def type_root(logical: str) -> str:
    """The logical type root of a Paimon SQL type name: "DECIMAL(10,2)" -> "DECIMAL", "INTEGER" -> "INT"."""
    root = logical.upper().split("(")[0].strip()
    return "INT" if root == "INTEGER" else root


def _type_args(logical: str) -> List[int]:
    if "(" not in logical:
        return []
    inner = logical[logical.index("(") + 1: logical.rindex(")")]
    return [int(a) for a in inner.split(",")]


def decimal_precision_scale(logical: str):
    """(precision, scale) of a DECIMAL type; DECIMAL alone is DECIMAL(10, 0) (DecimalType.java:41-45)."""
    args = _type_args(logical)
    precision = args[0] if args else 10
    scale = args[1] if len(args) > 1 else 0
    return precision, scale


def physical_type(logical: str) -> PhysicalType:
    root = type_root(logical)
    if root not in _LOGICAL:
        raise ValueError(f"unsupported type on the GPU merge path: {logical}")
    if root == "DECIMAL":
        p, s = decimal_precision_scale(logical)
        if not (1 <= p <= 18) or not (0 <= s <= p):
            raise ValueError(f"unsupported type on the GPU merge path: {logical} (DECIMAL is stored as an unscaled "
                             f"INT64: precision 1 to 18)")
    if root == "TIMESTAMP":
        args = _type_args(logical)
        if args and args[0] > 6:
            raise ValueError(f"unsupported type on the GPU merge path: {logical} (TIMESTAMP is stored as INT64 "
                             f"micros: precision up to 6)")
    return _LOGICAL[root]


# ORC TypeKind numbers (orc_proto Type.Kind) of the Paimon type roots, as OrcTypeUtil.convertToOrcType maps them
# (paimon-format/.../orc/OrcTypeUtil.java:50-120).  TIMESTAMP and CHAR are mapped too; the ORC encoder refuses them.
_ORC_KIND = {
    "BOOLEAN": 0, "TINYINT": 1, "SMALLINT": 2, "INT": 3, "TIME": 3, "BIGINT": 4, "FLOAT": 5, "DOUBLE": 6,
    "STRING": 7, "BINARY": 8, "VARBINARY": 8, "BYTES": 8, "TIMESTAMP": 9, "DECIMAL": 14, "DATE": 15, "VARCHAR": 16,
    "CHAR": 17,
}
VARCHAR_MAX_LENGTH = 2147483647            # VarCharType.MAX_LENGTH: STRING is VARCHAR of this length


def orc_column_type(logical: str):
    """(kind, precision, scale, max_length) of pg_orc_column_type for a Paimon SQL type name: DECIMAL keeps its
    precision and scale, VARCHAR(n) its length (VARCHAR of the maximum length is an ORC string)."""
    root = type_root(logical)
    if root not in _ORC_KIND:
        raise ValueError(f"unsupported type on the GPU merge path: {logical}")
    kind = _ORC_KIND[root]
    if root == "DECIMAL":
        p, s = decimal_precision_scale(logical)
        return kind, p, s, 0
    if root == "VARCHAR":
        args = _type_args(logical)
        n = args[0] if args else 1                   # VARCHAR alone is VARCHAR(1) (VarCharType.java)
        return (7, 0, 0, 0) if n == VARCHAR_MAX_LENGTH else (kind, 0, 0, n)
    return kind, 0, 0, 0


def numpy_dtype(t: PhysicalType):
    return _NP[PhysicalType(t)]


def is_varlen(t: PhysicalType) -> bool:
    return PhysicalType(t) in (PhysicalType.STRING, PhysicalType.BINARY)


@dataclass(frozen=True)
class DataField:
    name: str
    type: str            # Paimon SQL type name, e.g. "BIGINT", "VARCHAR(24)"
    nullable: bool = True

    @property
    def physical(self) -> PhysicalType:
        return physical_type(self.type)


@dataclass(frozen=True)
class RowType:
    fields: Sequence[DataField]

    def field_names(self) -> List[str]:
        return [f.name for f in self.fields]

    def index_of(self, name: str) -> int:
        return self.field_names().index(name)

    def __len__(self) -> int:
        return len(self.fields)


KEY_FIELD_PREFIX = "_KEY_"                 # SpecialFields.java:76
SEQUENCE_NUMBER = "_SEQUENCE_NUMBER"       # SpecialFields.java:79-80
VALUE_KIND = "_VALUE_KIND"                 # SpecialFields.java:82-83


@dataclass(frozen=True)
class KeyValueSchema:
    """File schema ``[_KEY_*…, _SEQUENCE_NUMBER BIGINT, _VALUE_KIND TINYINT, value…]``.

    Reference: KeyValue.schema (paimon-core/.../KeyValue.java:130-138) and
    PrimaryKeyTableUtils.addKeyNamePrefix (paimon-core/.../table/PrimaryKeyTableUtils.java:88-96).
    """

    key_type: RowType
    value_type: RowType

    @staticmethod
    def of(value_type: RowType, primary_keys: Sequence[str]) -> "KeyValueSchema":
        keys = []
        for pk in primary_keys:
            f = value_type.fields[value_type.index_of(pk)]
            keys.append(DataField(KEY_FIELD_PREFIX + f.name, f.type, False))
        return KeyValueSchema(RowType(tuple(keys)), value_type)

    @property
    def n_key(self) -> int:
        return len(self.key_type)

    @property
    def n_val(self) -> int:
        return len(self.value_type)

    @property
    def n_cols(self) -> int:
        return self.n_key + 2 + self.n_val

    def file_fields(self) -> List[DataField]:
        return (list(self.key_type.fields)
                + [DataField(SEQUENCE_NUMBER, "BIGINT", False), DataField(VALUE_KIND, "TINYINT", False)]
                + list(self.value_type.fields))

    def physical_types(self) -> List[PhysicalType]:
        return [f.physical for f in self.file_fields()]

    def decoded_bytes_per_row(self, mean_varlen: float = 16.0) -> float:
        """SURVEY §8(d): fixed width, var-len = 4-byte offset + payload, validity 1 bit/nullable cell."""
        total = 0.0
        for f in self.file_fields():
            t = f.physical
            total += (4 + mean_varlen) if is_varlen(t) else np.dtype(numpy_dtype(t)).itemsize
            if f.nullable:
                total += 1.0 / 8.0
        return total
