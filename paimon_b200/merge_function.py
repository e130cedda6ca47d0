"""Declarative mirror of the reference's ``MergeFunctionFactory`` family.

``MergeFunction`` is a per-record Java callback (reference:
paimon-core/src/main/java/org/apache/paimon/mergetree/compact/MergeFunction.java:37-53) and cannot
run on the device.  The factories below parse the *same* string-keyed table options the
reference factories parse and produce a ``MergeSpec`` — the plain struct that crosses the C ABI
(``pg_merge_spec`` in include/paimon_gpu.h).  Specs the device path does not implement are
refused here, at plan time; there is no CPU fallback.

Option parsing follows:
  DeduplicateMergeFunction.factory            (…/compact/DeduplicateMergeFunction.java:66-90)
  PartialUpdateMergeFunction.Factory          (…/compact/PartialUpdateMergeFunction.java:389-489, 657-687)
  AggregateMergeFunction.Factory/getAggFuncName (…/compact/aggregate/AggregateMergeFunction.java:146-204)
  FieldAggregatorFactory.create               (…/compact/aggregate/factory/FieldAggregatorFactory.java:39-65)
  CoreOptions keys                            (paimon-api/.../CoreOptions.java:72-79, 585, 955-986, 1929)
"""
from __future__ import annotations

import enum
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

from .types import DataField, KeyValueSchema, RowType, decimal_precision_scale, type_root


class MergeEngine(enum.IntEnum):          # CoreOptions.MergeEngine (CoreOptions.java:3910-3917)
    DEDUPLICATE = 0
    PARTIAL_UPDATE = 1
    AGGREGATE = 2
    FIRST_ROW = 3


class SortEngine(enum.IntEnum):           # CoreOptions.SortEngine (CoreOptions.java:4228-4232)
    LOSER_TREE = 0
    MIN_HEAP = 1


class Agg(enum.IntEnum):
    NONE = 0
    SUM = 1
    PRODUCT = 2
    MAX = 3
    MIN = 4
    BOOL_AND = 5
    BOOL_OR = 6
    LAST_VALUE = 7
    LAST_NON_NULL_VALUE = 8
    FIRST_VALUE = 9
    FIRST_NON_NULL_VALUE = 10
    PRIMARY_KEY = 11


_AGG_NAMES = {
    "sum": Agg.SUM, "product": Agg.PRODUCT, "max": Agg.MAX, "min": Agg.MIN,
    "bool_and": Agg.BOOL_AND, "bool_or": Agg.BOOL_OR, "last_value": Agg.LAST_VALUE,
    "last_non_null_value": Agg.LAST_NON_NULL_VALUE, "first_value": Agg.FIRST_VALUE,
    "first_non_null_value": Agg.FIRST_NON_NULL_VALUE, "primary-key": Agg.PRIMARY_KEY,
}
# aggregators with variable-size object state; refused at plan time (SURVEY §2.2)
_UNSUPPORTED_AGGS = {"listagg", "collect", "merge_map", "merge_map_with_keytime", "nested_update",
                     "nested_partial_update", "theta_sketch", "hll_sketch", "rbm32", "rbm64"}

FIELDS_PREFIX = "fields"
AGG_FUNCTION = "aggregate-function"
DEFAULT_AGG_FUNCTION = "default-aggregate-function"
IGNORE_RETRACT = "ignore-retract"
SEQUENCE_GROUP = "sequence-group"


class UnsupportedMergeSpec(ValueError):
    """Raised at plan time for a spec the device path refuses (no CPU fallback)."""


def _bool(v) -> bool:
    return str(v).strip().lower() == "true" if not isinstance(v, bool) else v


@dataclass
class MergeSpec:
    """What the native library needs to know about the merge; one per reader."""

    engine: MergeEngine = MergeEngine.DEDUPLICATE
    ignore_delete: bool = False
    remove_record_on_delete: bool = False
    drop_delete: bool = False                       # DropDeleteReader wrapped around the merge
    seq_fields: List[int] = field(default_factory=list)   # 'sequence.field' as value-field indexes
    seq_ascending: bool = True
    agg: List[Agg] = field(default_factory=list)           # per value field
    ignore_retract: List[bool] = field(default_factory=list)
    groups: List[List[int]] = field(default_factory=list)  # sequence fields of each sequence group
    field_group: List[int] = field(default_factory=list)   # per value field: protecting group or -1
    group_partial_delete: List[bool] = field(default_factory=list)
    # read-type projection (MergeFunctionFactory.create(readType)): per value field, part of the merged batch;
    # empty = every field.  Field indexes everywhere in the spec stay those of the table's row type.
    read_fields: List[bool] = field(default_factory=list)
    # per value field: precision << 8 | scale of a DECIMAL field, 0 for every other type; empty = no DECIMAL field.
    # SUM / PRODUCT on a DECIMAL field follow DecimalUtils / BigDecimal, not int64 arithmetic on the unscaled value.
    decimal: List[int] = field(default_factory=list)

    def with_read_fields(self, mask: Sequence[bool]) -> "MergeSpec":
        import copy
        s = copy.deepcopy(self)
        s.read_fields = [bool(b) for b in mask]
        return s

    def fields_the_merge_reads(self, n_val: int) -> List[bool]:
        """Value fields a reader has to decode for this spec: the read type plus what the merge function itself
        compares — 'sequence.field' columns and every sequence-group field (PartialUpdateMergeFunction.adjustReadType,
        PartialUpdateMergeFunction.java:576-606)."""
        need = list(self.read_fields) if self.read_fields else [True] * n_val
        for f in self.seq_fields:
            need[f] = True
        for g in self.groups:
            for f in g:
                need[f] = True
        return need

    def with_drop_delete(self, drop: bool = True) -> "MergeSpec":
        import copy
        s = copy.deepcopy(self)
        s.drop_delete = drop
        return s

    def normalised(self, n_val: int) -> "MergeSpec":
        import copy
        s = copy.deepcopy(self)
        s.agg = list(s.agg) or [Agg.NONE] * n_val
        s.ignore_retract = list(s.ignore_retract) or [False] * n_val
        s.field_group = list(s.field_group) or [-1] * n_val
        s.group_partial_delete = list(s.group_partial_delete) or [False] * n_val
        return s


class MergeFunctionFactory:
    """Mirror of MergeFunctionFactory.create(readType) (…/compact/MergeFunctionFactory.java:29-41)."""

    def create(self, read_type: Optional[RowType] = None) -> MergeSpec:
        raise NotImplementedError


def _sequence_fields(options: Dict[str, str], row_type: RowType):
    raw = options.get("sequence.field")
    names = [s.strip() for s in raw.split(",")] if raw else []
    asc = options.get("sequence.field.sort-order", "ascending").lower() == "ascending"
    return [row_type.index_of(n) for n in names], names, asc


# logical type roots of the NUMERIC family (DataTypeRoot.java), the only ones FieldSumAggFactory /
# FieldProductAggFactory accept
_NUMERIC_ROOTS = {"TINYINT", "SMALLINT", "INT", "BIGINT", "FLOAT", "DOUBLE", "DECIMAL"}
# roots InternalRowUtils.compare orders (InternalRowUtils.java:387-432), what FieldMaxAgg / FieldMinAgg need
_COMPARABLE_ROOTS = _NUMERIC_ROOTS | {"DATE", "TIME", "TIMESTAMP", "CHAR", "VARCHAR", "STRING", "BINARY",
                                      "VARBINARY", "BYTES"}


def _resolve_agg(name: str, f: DataField) -> Agg:
    """FieldAggregatorFactory.create: the aggregator's factory checks the field's LOGICAL type root
    (FieldSumAggFactory.java:33-39, FieldProductAggFactory.java:33-39, FieldBoolAndAggFactory.java:33-39)."""
    if name in _UNSUPPORTED_AGGS:
        raise UnsupportedMergeSpec(
            f"aggregate function '{name}' on field '{f.name}' keeps variable-size state and is "
            f"not implemented on the device merge path")
    if name not in _AGG_NAMES:
        raise ValueError(f"Use unsupported aggregation: {name} or spell aggregate function incorrectly!")
    agg = _AGG_NAMES[name]
    f.physical                                                  # refuses types the device cannot store
    root = type_root(f.type)
    if agg in (Agg.SUM, Agg.PRODUCT) and root not in _NUMERIC_ROOTS:
        raise ValueError(f"Data type for {name} column must be 'NumericType' but was '{f.type}'.")
    if agg in (Agg.BOOL_AND, Agg.BOOL_OR) and root != "BOOLEAN":
        raise ValueError(f"Data type for {name.replace('_', ' ')} column must be 'BooleanType' but was '{f.type}'.")
    if agg in (Agg.MAX, Agg.MIN) and root not in _COMPARABLE_ROOTS:
        raise ValueError(f"Incomparable type: {f.type}")                     # InternalRowUtils.compare
    return agg


def decimal_descriptors(row_type: RowType) -> List[int]:
    """MergeSpec.decimal of a row type: precision << 8 | scale per DECIMAL field, 0 elsewhere; empty when the row has
    no DECIMAL field."""
    out = []
    for f in row_type.fields:
        if type_root(f.type) == "DECIMAL":
            p, s = decimal_precision_scale(f.type)
            out.append(p << 8 | s)
        else:
            out.append(0)
    return out if any(out) else []


class DeduplicateMergeFunction:
    @staticmethod
    def factory(options: Optional[Dict[str, str]] = None) -> MergeFunctionFactory:
        ignore_delete = _bool((options or {}).get("ignore-delete", False))

        class _F(MergeFunctionFactory):
            def create(self, read_type=None) -> MergeSpec:
                return MergeSpec(engine=MergeEngine.DEDUPLICATE, ignore_delete=ignore_delete)
        return _F()


class FirstRowMergeFunction:
    @staticmethod
    def factory(options: Optional[Dict[str, str]] = None) -> MergeFunctionFactory:
        ignore_delete = _bool((options or {}).get("ignore-delete", False))

        class _F(MergeFunctionFactory):
            def create(self, read_type=None) -> MergeSpec:
                return MergeSpec(engine=MergeEngine.FIRST_ROW, ignore_delete=ignore_delete)
        return _F()


class AggregateMergeFunction:
    @staticmethod
    def factory(options: Dict[str, str], row_type: RowType, primary_keys: Sequence[str]) -> MergeFunctionFactory:
        options = dict(options or {})

        class _F(MergeFunctionFactory):
            def create(self, read_type=None) -> MergeSpec:
                target = read_type or row_type
                _, seq_names, _ = _sequence_fields(options, target) if options.get("sequence.field") else ([], [], True)
                aggs, ign = [], []
                for f in target.fields:
                    # getAggFuncName, AggregateMergeFunction.java:179-204
                    if f.name in seq_names:
                        name = "last_value"
                    elif f.name in primary_keys:
                        name = "primary-key"
                    else:
                        name = (options.get(f"{FIELDS_PREFIX}.{f.name}.{AGG_FUNCTION}")
                                or options.get(f"{FIELDS_PREFIX}.{DEFAULT_AGG_FUNCTION}")
                                or "last_non_null_value")
                    aggs.append(_resolve_agg(name, f))
                    ign.append(_bool(options.get(f"{FIELDS_PREFIX}.{f.name}.{IGNORE_RETRACT}", False)))
                return MergeSpec(engine=MergeEngine.AGGREGATE,
                                 remove_record_on_delete=_bool(options.get("aggregation.remove-record-on-delete", False)),
                                 agg=aggs, ignore_retract=ign, decimal=decimal_descriptors(target))
        return _F()


class PartialUpdateMergeFunction:
    @staticmethod
    def factory(options: Dict[str, str], row_type: RowType, primary_keys: Sequence[str]) -> MergeFunctionFactory:
        options = dict(options or {})
        ignore_delete = _bool(options.get("ignore-delete", False))
        remove_on_delete = _bool(options.get("partial-update.remove-record-on-delete", False))
        remove_on_group = options.get("partial-update.remove-record-on-sequence-group")
        names = row_type.field_names()

        def require(fname: str) -> int:
            if fname not in names:
                raise ValueError(f"Field {fname} can not be found in table schema")
            return names.index(fname)

        groups: List[List[int]] = []
        field_group = [-1] * len(names)
        all_sequence_fields: List[str] = []
        protected: List[str] = []
        seq_group_of: Dict[str, int] = {}
        for k, v in options.items():                           # :400-445
            if k.startswith(FIELDS_PREFIX + ".") and k.endswith("." + SEQUENCE_GROUP):
                seq_names = k[len(FIELDS_PREFIX) + 1: len(k) - len(SEQUENCE_GROUP) - 1].split(",")
                seq_idx = [require(n.strip()) for n in seq_names]
                gid = len(groups)
                groups.append(seq_idx)
                for fname in v.split(","):
                    fi = require(fname.strip())
                    if field_group[fi] != -1:
                        raise ValueError(f"Field {names[fi]} is defined repeatedly by multiple groups: {k}")
                    field_group[fi] = gid
                    protected.append(names[fi])
                for fi in seq_idx:
                    all_sequence_fields.append(names[fi])
                    field_group[fi] = gid
                    seq_group_of[names[fi]] = fi
        if remove_on_delete and ignore_delete:
            raise ValueError("ignore-delete and partial-update.remove-record-on-delete have conflicting "
                             "behavior so should not be enabled at the same time.")
        if remove_on_group is not None and ignore_delete:
            raise ValueError("ignore-delete and partial-update.remove-record-on-sequence-group have "
                             "conflicting behavior so should not be enabled at the same time.")
        if remove_on_delete and groups:
            raise ValueError("sequence-group and partial-update.remove-record-on-delete have conflicting "
                             "behavior so should not be enabled at the same time.")
        partial_delete = [False] * len(names)
        if remove_on_group is not None:
            for fname in remove_on_group.split(","):
                if fname not in seq_group_of:
                    raise ValueError(f"field '{remove_on_group}' defined in "
                                     f"'partial-update.remove-record-on-sequence-group' option must be part "
                                     f"of sequence groups")
                partial_delete[seq_group_of[fname]] = True

        aggs = []
        ign = []
        for f in row_type.fields:                              # getAggFuncName :657-687
            if f.name in all_sequence_fields:
                name = None
            elif f.name in primary_keys:
                name = "primary-key"
            else:
                name = (options.get(f"{FIELDS_PREFIX}.{f.name}.{AGG_FUNCTION}")
                        or options.get(f"{FIELDS_PREFIX}.{DEFAULT_AGG_FUNCTION}"))
                if name is not None and name != "last_non_null_value" and f.name not in protected:
                    raise ValueError(f"Must use sequence group for aggregation functions but not found "
                                     f"for field {f.name}.")
            aggs.append(Agg.NONE if name is None else _resolve_agg(name, f))
            ign.append(_bool(options.get(f"{FIELDS_PREFIX}.{f.name}.{IGNORE_RETRACT}", False)))

        class _F(MergeFunctionFactory):
            def create(self, read_type=None) -> MergeSpec:
                spec = MergeSpec(engine=MergeEngine.PARTIAL_UPDATE, ignore_delete=ignore_delete,
                                 remove_record_on_delete=remove_on_delete, agg=list(aggs),
                                 ignore_retract=list(ign), groups=[list(g) for g in groups],
                                 field_group=list(field_group), group_partial_delete=list(partial_delete),
                                 decimal=decimal_descriptors(row_type))
                if read_type is not None and read_type.field_names() != names:
                    # a projected read type (PartialUpdateMergeFunction.java:492-573 re-indexes the per-field
                    # configuration; here the indexes stay those of the table and the projection is a mask)
                    unknown = [n for n in read_type.field_names() if n not in names]
                    if unknown:
                        raise ValueError(f"read type has fields the table does not have: {unknown}")
                    wanted = set(read_type.field_names())
                    spec.read_fields = [n in wanted for n in names]
                return spec
        return _F()


def merge_function_factory(options: Dict[str, str], row_type: RowType, primary_keys: Sequence[str]) -> MergeFunctionFactory:
    """PrimaryKeyTableUtils.createMergeFunctionFactory (paimon-core/.../table/PrimaryKeyTableUtils.java:62-86)."""
    engine = (options or {}).get("merge-engine", "deduplicate")
    if engine == "deduplicate":
        return DeduplicateMergeFunction.factory(options)
    if engine == "partial-update":
        return PartialUpdateMergeFunction.factory(options, row_type, primary_keys)
    if engine == "aggregation":
        return AggregateMergeFunction.factory(options, row_type, primary_keys)
    if engine == "first-row":
        return FirstRowMergeFunction.factory(options)
    raise ValueError(f"Unsupported merge engine: {engine}")


class UserDefinedSeqComparator:
    """Mirror of paimon-core/.../utils/UserDefinedSeqComparator.java:30-96: the 'sequence.field' columns and their
    sort order.  On the device it is data (field indexes + order), not code."""

    def __init__(self, fields: Sequence[int], ascending: bool = True):
        self.fields = list(fields)
        self.ascending = bool(ascending)

    def compare_fields(self) -> List[int]:
        return list(self.fields)

    def is_ascending_order(self) -> bool:
        return self.ascending

    @staticmethod
    def create(row_type: RowType, options: Dict[str, str]) -> Optional["UserDefinedSeqComparator"]:
        """UserDefinedSeqComparator.create(rowType, CoreOptions): None when 'sequence.field' is not set."""
        raw = (options or {}).get("sequence.field")
        if not raw:
            return None
        fields = [row_type.index_of(n.strip()) for n in raw.split(",")]
        asc = (options or {}).get("sequence.field.sort-order", "ascending").lower() == "ascending"
        return UserDefinedSeqComparator(fields, asc)

    def apply(self, spec: "MergeSpec") -> "MergeSpec":
        import copy
        s = copy.deepcopy(spec)
        s.seq_fields = list(self.fields)
        s.seq_ascending = self.ascending
        return s
