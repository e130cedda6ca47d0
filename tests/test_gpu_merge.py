"""Parity of the CUDA merge path (through the C ABI) against the CPU oracle.  Needs an H100."""
import random

import numpy as np
import pytest

from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.merge_function import (AggregateMergeFunction, DeduplicateMergeFunction,
                                        FirstRowMergeFunction, PartialUpdateMergeFunction)
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader, merge_runs
from paimon_b200.types import DataField, KeyValueSchema, RowKind, RowType

from reusing_test_data import SCHEMA, VALUE_TYPE, generate_random_readers, parse, to_batch
from test_oracle_golden import FIXED_VECTORS

pytestmark = pytest.mark.gpu


def assert_same(schema, spec, runs):
    want = pyoracle.merge(schema, spec, runs, pyoracle.SORT_LOSER_TREE)
    got = merge_runs(schema, spec, runs)
    assert got.equals(want), got.first_difference(want)
    return got


SPECS = {
    "dedup": DeduplicateMergeFunction.factory().create(),
    "dedup_ignore_delete": DeduplicateMergeFunction.factory({"ignore-delete": "true"}).create(),
    "dedup_drop_delete": DeduplicateMergeFunction.factory().create().with_drop_delete(),
    "first_row_ignore_delete": FirstRowMergeFunction.factory({"ignore-delete": "true"}).create(),
    "pu_ignore_delete": PartialUpdateMergeFunction.factory({"ignore-delete": "true"}, VALUE_TYPE, ["f0"]).create(),
    "pu_remove_on_delete": PartialUpdateMergeFunction.factory(
        {"partial-update.remove-record-on-delete": "true"}, VALUE_TYPE, ["f0"]).create(),
    "agg_sum": AggregateMergeFunction.factory({"fields.f1.aggregate-function": "sum"}, VALUE_TYPE, ["f0"]).create(),
    "agg_sum_remove_on_delete": AggregateMergeFunction.factory(
        {"fields.f1.aggregate-function": "sum", "aggregation.remove-record-on-delete": "true"},
        VALUE_TYPE, ["f0"]).create(),
    "agg_default": AggregateMergeFunction.factory({}, VALUE_TYPE, ["f0"]).create(),
    "agg_max_ignore_retract": AggregateMergeFunction.factory(
        {"fields.f1.aggregate-function": "max", "fields.f1.ignore-retract": "true"}, VALUE_TYPE, ["f0"]).create(),
    "agg_product_drop_delete": AggregateMergeFunction.factory(
        {"fields.f1.aggregate-function": "product"}, VALUE_TYPE, ["f0"]).create().with_drop_delete(),
}


@pytest.mark.parametrize("spec_name", sorted(SPECS))
@pytest.mark.parametrize("name", sorted(FIXED_VECTORS))
def test_fixed_vectors(name, spec_name):
    readers = [to_batch(parse(s)) for s in FIXED_VECTORS[name]]
    assert_same(SCHEMA, SPECS[spec_name], readers)


@pytest.mark.parametrize("spec_name", sorted(SPECS))
def test_random_rounds(spec_name):
    """CombiningRecordReaderTestBase.testRandom (1-20 readers x 1-100 rows), every engine."""
    rng = random.Random(hash(spec_name) & 0xffff)
    for _ in range(25):
        readers = [to_batch(r) for r in generate_random_readers(rng, only_add=False)]
        assert_same(SCHEMA, SPECS[spec_name], readers)


def test_first_row_add_only_and_error():
    rng = random.Random(3)
    spec = FirstRowMergeFunction.factory().create()
    for _ in range(10):
        readers = [to_batch(r) for r in generate_random_readers(rng, only_add=True)]
        assert_same(SCHEMA, spec, readers)
    readers = [to_batch(parse("1, 1, +, 10")), to_batch(parse("1, 3, -, 11"))]
    with pytest.raises(N.MergeFunctionError, match="First row merge engine can not accept"):
        merge_runs(SCHEMA, spec, readers)


def test_partial_update_delete_error_message():
    spec = PartialUpdateMergeFunction.factory({}, VALUE_TYPE, ["f0"]).create()
    readers = [to_batch(parse("1, 1, +, 10")), to_batch(parse("1, 3, -, 11"))]
    with pytest.raises(N.MergeFunctionError, match="Partial update can not accept delete records"):
        merge_runs(SCHEMA, spec, readers)
    # a lone DELETE passes through untouched (ReducerMergeFunctionWrapper)
    got = merge_runs(SCHEMA, spec, [to_batch(parse("1, 3, -, 11"))])
    assert got.to_rows() == [(1, 3, 3, 1, 11)]


def test_agg_retract_unsupported_error():
    spec = AggregateMergeFunction.factory({"fields.f1.aggregate-function": "max"}, VALUE_TYPE, ["f0"]).create()
    readers = [to_batch(parse("1, 1, +, 10")), to_batch(parse("1, 3, -, 11"))]
    with pytest.raises(N.MergeFunctionError, match="does not support retraction"):
        merge_runs(SCHEMA, spec, readers)


def test_unsupported_specs_are_refused():
    # DOUBLE primary key (NaN compares equal to everything in the reference): refused at plan time, no CPU fallback
    vt = RowType((DataField("k", "DOUBLE", False), DataField("v", "BIGINT", True)))
    schema = KeyValueSchema.of(vt, ["k"])
    run = KeyValueBatch.from_rows(schema, [(1.0, 1, 0, 1.0, 5)])
    with pytest.raises(N.UnsupportedOnDevice):
        merge_runs(schema, DeduplicateMergeFunction.factory().create(), [run, run])


def test_empty_and_single_inputs():
    spec = DeduplicateMergeFunction.factory().create()
    assert merge_runs(SCHEMA, spec, []).n_rows == 0
    assert merge_runs(SCHEMA, spec, [to_batch([])]).n_rows == 0
    assert merge_runs(SCHEMA, spec, [to_batch([]), to_batch([]), to_batch([])]).n_rows == 0
    one = to_batch(parse("1, 1, +, 100 | 2, 500, -, 200"))
    assert_same(SCHEMA, spec, [one])
    rd = SortMergeReader.create_sort_merge_reader([SortedRunReader(SCHEMA, to_batch([]))], None, None, spec)
    assert rd.read_batch() is None
    rd.close()


def all_types_schema():
    vt = RowType((DataField("pk", "INT", False), DataField("t", "TINYINT", True), DataField("s", "SMALLINT", True),
                  DataField("i", "INT", True), DataField("l", "BIGINT", True), DataField("f", "FLOAT", True),
                  DataField("d", "DOUBLE", True), DataField("b", "BOOLEAN", True), DataField("str", "STRING", True),
                  DataField("bin", "BINARY", True), DataField("nn", "BIGINT", False)))
    return KeyValueSchema.of(vt, ["pk"]), vt


def random_all_types_runs(rng, n_runs, max_rows, key_space, kinds):
    schema, _ = all_types_schema()
    runs, seq = [], 0
    for r in range(n_runs):
        n = rng.randrange(0, max_rows + 1)
        keys = sorted(rng.sample(range(key_space), min(n, key_space)))
        rows = []
        for k in keys:
            seq += rng.randrange(1, 5)
            def opt(v):
                return None if rng.random() < 0.3 else v
            rows.append((k, seq * 7919 % 100003 + seq, rng.choice(kinds), k,
                         opt(rng.randrange(-128, 128)), opt(rng.randrange(-32768, 32768)),
                         opt(rng.randrange(-2 ** 31, 2 ** 31)), opt(rng.randrange(-2 ** 63, 2 ** 63)),
                         opt(rng.uniform(-1e3, 1e3)), opt(rng.uniform(-1e6, 1e6)), opt(rng.randrange(2)),
                         opt("".join(rng.choice("abcxyz") for _ in range(rng.randrange(0, 12)))),
                         opt(bytes(rng.randrange(256) for _ in range(rng.randrange(0, 9)))),
                         rng.randrange(-1000, 1000)))
        runs.append(KeyValueBatch.from_rows(schema, rows))
    return schema, runs


ALL_TYPES_SPECS = {
    "dedup": lambda vt: DeduplicateMergeFunction.factory().create(),
    "pu": lambda vt: PartialUpdateMergeFunction.factory({"ignore-delete": "true"}, vt, ["pk"]).create(),
    "pu_rod": lambda vt: PartialUpdateMergeFunction.factory({"partial-update.remove-record-on-delete": "true"}, vt, ["pk"]).create(),
    "agg_mixed": lambda vt: AggregateMergeFunction.factory({
        "fields.t.aggregate-function": "sum", "fields.s.aggregate-function": "product",
        "fields.i.aggregate-function": "max", "fields.l.aggregate-function": "sum",
        "fields.f.aggregate-function": "sum", "fields.d.aggregate-function": "sum",
        "fields.b.aggregate-function": "bool_or", "fields.str.aggregate-function": "max",
        "fields.bin.aggregate-function": "first_non_null_value", "fields.nn.aggregate-function": "min",
        "fields.i.ignore-retract": "true", "fields.b.ignore-retract": "true", "fields.str.ignore-retract": "true",
        "fields.bin.ignore-retract": "true", "fields.nn.ignore-retract": "true"}, vt, ["pk"]).create(),
    "agg_first_last": lambda vt: AggregateMergeFunction.factory({
        "fields.default-aggregate-function": "first_value", "fields.l.aggregate-function": "last_value",
        "fields.d.aggregate-function": "product", "fields.str.aggregate-function": "min",
        "fields.f.aggregate-function": "min", "fields.b.aggregate-function": "bool_and"}, vt, ["pk"]).create(),
}


@pytest.mark.parametrize("spec_name", sorted(ALL_TYPES_SPECS))
def test_all_types_nulls_varlen(spec_name):
    """35-type-row spirit of ParquetReadWriteTest / FieldAggregatorTest: every physical type, 30 % nulls,
    var-len columns, retract rows where the spec tolerates them."""
    rng = random.Random(17)
    _, vt = all_types_schema()
    spec = ALL_TYPES_SPECS[spec_name](vt)
    kinds = [0, 0, 0, 2] if spec_name == "agg_first_last" else [0, 0, 2, 3, 1]
    for _ in range(12):
        schema, runs = random_all_types_runs(rng, rng.randrange(1, 9), 60, 90, kinds)
        assert_same(schema, spec, runs)


@pytest.mark.parametrize("n_runs,total", [(2, 20000), (8, 100000), (16, 300000), (32, 200000)])
def test_multi_tile_deduplicate(n_runs, total):
    """Large enough for several partition levels (tiles of <= 4096 rows, stride-32 sampling)."""
    schema = datagen.schema_c2()
    runs = datagen.make_runs(schema, n_runs, total, seed=3, null_prob=0.2, delete_prob=0.05)
    got = assert_same(schema, DeduplicateMergeFunction.factory().create(), runs)
    keys = got.columns[0].data
    assert np.all(keys[1:] > keys[:-1])          # strictly increasing keys: sorted and deduplicated


def test_multi_tile_partial_update_wide_row():
    schema = datagen.schema_c3(n_i64=4, n_f64=3, n_str=3)
    runs = datagen.make_runs(schema, 16, 120000, seed=5, null_prob=0.5)
    spec = PartialUpdateMergeFunction.factory({}, schema.value_type, ["pk"]).create()
    assert_same(schema, spec, runs)


@pytest.mark.parametrize("engine", ["partial-update", "deduplicate"])
def test_more_than_64_select_columns(engine):
    """The emit kernel resolves select columns through per-member take masks of 64 columns: a 100-column row
    needs two passes over the column chunks."""
    schema = datagen.schema_c3(n_i64=60, n_f64=25, n_str=14)
    runs = datagen.make_runs(schema, 6, 30000, seed=11, null_prob=0.5, delete_prob=0.05 if engine == "deduplicate" else 0.0)
    if engine == "partial-update":
        spec = PartialUpdateMergeFunction.factory({}, schema.value_type, ["pk"]).create()
    else:
        spec = DeduplicateMergeFunction.factory().create()
    assert_same(schema, spec, runs)


def test_multi_tile_aggregate_double_sum_is_bit_exact():
    schema = datagen.schema_c3(n_i64=2, n_f64=4, n_str=1)
    runs = datagen.make_runs(schema, 16, 100000, seed=9, null_prob=0.3)
    opts = {f"fields.d{i}.aggregate-function": "sum" for i in range(4)}
    opts["fields.i0.aggregate-function"] = "sum"
    spec = AggregateMergeFunction.factory(opts, schema.value_type, ["pk"]).create()
    assert_same(schema, spec, runs)


def test_skewed_run_lengths_and_tiny_runs():
    schema = datagen.schema_c1()
    rng = np.random.default_rng(0)
    sizes = [50000, 3, 0, 17000, 1, 31, 33, 4097]
    runs = [datagen.make_run(schema, r, datagen.run_keys(rng, 40000, n), seed=2) for r, n in enumerate(sizes)]
    assert_same(schema, DeduplicateMergeFunction.factory().create(), runs)


def test_composite_and_narrow_keys():
    vt = RowType((DataField("a", "INT", False), DataField("b", "SMALLINT", False), DataField("v", "BIGINT", True)))
    schema = KeyValueSchema.of(vt, ["a", "b"])
    rng = random.Random(8)
    runs, seq = [], 0
    for r in range(5):
        keys = sorted({(rng.randrange(-50, 50), rng.randrange(-3, 3)) for _ in range(300)})
        rows = []
        for (a, b) in keys:
            seq += 1
            rows.append((a, b, seq, 0, a, b, rng.randrange(100)))
        runs.append(KeyValueBatch.from_rows(schema, rows))
    assert_same(schema, DeduplicateMergeFunction.factory().create(), runs)


def test_size_independent_properties_at_scale():
    """C1-shaped 2M rows: checks that do not need the oracle — sortedness, idempotence, row conservation."""
    schema = datagen.schema_c1()
    runs = datagen.make_runs(schema, 4, 2_000_000, seed=11)
    spec = DeduplicateMergeFunction.factory().create()
    got = merge_runs(schema, spec, runs)
    keys = got.columns[0].data
    assert np.all(keys[1:] > keys[:-1])
    all_keys = np.concatenate([r.columns[0].data for r in runs])
    assert got.n_rows == len(np.unique(all_keys))
    # the winner of every key is the row with the highest sequence number
    all_seq = np.concatenate([r.sequence_numbers for r in runs])
    order = np.lexsort((all_seq, all_keys))
    last = np.r_[all_keys[order][1:] != all_keys[order][:-1], True]
    assert np.array_equal(got.sequence_numbers, all_seq[order][last])
    # merging the merged result with nothing changes nothing
    again = merge_runs(schema, spec, [got])
    assert again.equals(got)


@pytest.mark.parametrize("ascending", [True, False])
@pytest.mark.parametrize("engine", ["dedup", "partial-update", "aggregation"])
def test_user_defined_sequence_fields(engine, ascending):
    """'sequence.field': members are ordered by the user fields (nulls first, before the descending flip;
    GenerateUtils.scala:305-345), then by _SEQUENCE_NUMBER (SortMergeReaderWithLoserTree.java:58-64)."""
    from paimon_b200.merge_function import UserDefinedSeqComparator
    vt = RowType((DataField("pk", "INT", False), DataField("ts", "INT", True), DataField("score", "DOUBLE", True),
                  DataField("v", "BIGINT", True), DataField("s", "STRING", True)))
    schema = KeyValueSchema.of(vt, ["pk"])
    opts = {"sequence.field": "ts,score", "sequence.field.sort-order": "ascending" if ascending else "descending"}
    if engine == "dedup":
        spec = DeduplicateMergeFunction.factory(opts).create()
    elif engine == "partial-update":
        spec = PartialUpdateMergeFunction.factory(opts, vt, ["pk"]).create()
    else:
        spec = AggregateMergeFunction.factory(dict(opts, **{"fields.v.aggregate-function": "sum"}), vt, ["pk"]).create()
    udsc = UserDefinedSeqComparator.create(vt, opts)
    assert udsc.compare_fields() == [1, 2] and udsc.is_ascending_order() == ascending
    rng = random.Random(77 + ascending)
    for _ in range(10):
        runs, seq = [], 0
        for r in range(rng.randrange(2, 9)):
            keys = sorted(rng.sample(range(60), rng.randrange(1, 50)))
            rows = []
            for kx in keys:
                seq += 1
                rows.append((kx, seq, 0, kx,
                             None if rng.random() < 0.3 else rng.randrange(0, 4),          # many ties and nulls
                             None if rng.random() < 0.3 else rng.choice([1.5, 2.5, float("nan"), -0.0, 0.0]),
                             None if rng.random() < 0.2 else rng.randrange(-1000, 1000),
                             None if rng.random() < 0.3 else rng.choice(["a", "bb", "ccc"])))
            runs.append(KeyValueBatch.from_rows(schema, rows))
        want = pyoracle.merge(schema, udsc.apply(spec), runs, pyoracle.SORT_LOSER_TREE)
        readers = [SortedRunReader(schema, b) for b in runs]
        rd = SortMergeReader.create_sort_merge_reader(readers, None, udsc, spec)
        try:
            rd.execute()
            got = rd.fetch()
        finally:
            rd.close()
        assert got.equals(want), got.first_difference(want)


def _utf8_sort_key(x):
    return x.encode() if isinstance(x, str) else x


@pytest.mark.parametrize("case", ["short_strings", "long_common_prefix", "prefix_of_each_other", "binary_high_bytes",
                                  "string_then_int", "bigint_then_int", "int_then_string"])
def test_general_primary_keys(case):
    """Keys that do not fit the 64-bit prefix exactly: strings / binaries (unsigned bytewise, then length —
    BinaryString.java:109-126, SortUtil.java:212-241) and wide composites; ties on the prefix are resolved by the
    full comparison."""
    rng = random.Random(hash(case) & 0xffff)
    if case in ("short_strings", "long_common_prefix", "prefix_of_each_other"):
        vt = RowType((DataField("k", "STRING", False), DataField("v", "BIGINT", True)))
        pk = ["k"]
        if case == "short_strings":
            mk = lambda rng: "".join(rng.choice("abc") for _ in range(rng.randrange(0, 6)))
        elif case == "long_common_prefix":
            mk = lambda rng: "customer_id_000000_" + "%06d" % rng.randrange(3000)
        else:
            mk = lambda rng: "ab" * rng.randrange(0, 9) + rng.choice(["", "\x00", "\x01", "a"])
        sort = lambda u: sorted(u, key=_utf8_sort_key)
    elif case == "binary_high_bytes":
        vt = RowType((DataField("k", "BINARY", False), DataField("v", "BIGINT", True)))
        pk = ["k"]
        mk = lambda rng: bytes(rng.choice([0, 1, 127, 128, 255]) for _ in range(rng.randrange(0, 12)))
        sort = sorted
    elif case == "string_then_int":
        vt = RowType((DataField("s", "STRING", False), DataField("i", "INT", False), DataField("v", "BIGINT", True)))
        pk = ["s", "i"]
        mk = lambda rng: (rng.choice(["", "a", "ab", "abcdefgh", "abcdefghi", "b"]), rng.randrange(-3, 3))
        sort = lambda u: sorted(u, key=lambda t: (t[0].encode(), t[1]))
    elif case == "bigint_then_int":
        vt = RowType((DataField("o", "BIGINT", False), DataField("l", "INT", False), DataField("v", "BIGINT", True)))
        pk = ["o", "l"]
        mk = lambda rng: (rng.choice([-2 ** 63, -5, 0, 7, 2 ** 40, 2 ** 63 - 1]) + rng.randrange(0, 3) * 0, rng.randrange(-4, 4))
        sort = sorted
    else:
        vt = RowType((DataField("i", "INT", False), DataField("s", "STRING", False), DataField("v", "BIGINT", True)))
        pk = ["i", "s"]
        mk = lambda rng: (rng.randrange(-2, 3), "".join(rng.choice("xyz") for _ in range(rng.randrange(0, 10))))
        sort = lambda u: sorted(u, key=lambda t: (t[0], t[1].encode()))
    schema = KeyValueSchema.of(vt, pk)
    for n_runs, n_keys in ((2, 40), (7, 300), (16, 6000)):
        universe = sort({mk(rng) for _ in range(n_keys)})
        runs, seq = [], 0
        for r in range(n_runs):
            rows = []
            for key in universe:
                if rng.random() < 0.4:
                    seq += 1
                    kt = key if isinstance(key, tuple) else (key,)
                    rows.append(kt + (seq, rng.choice([0, 0, 0, 3])) + kt + (rng.randrange(1000),))
            runs.append(KeyValueBatch.from_rows(schema, rows))
        assert_same(schema, DeduplicateMergeFunction.factory().create(), runs)
        assert_same(schema, AggregateMergeFunction.factory({"fields.v.aggregate-function": "sum",
                                                           "fields.v.ignore-retract": "true"}, vt, pk).create(), runs)


# ---------------------------------------------------------------- partial-update sequence groups

class GpuFuncDriver:
    """PartialUpdateMergeFunctionTest-style driver on the device: after n >= 2 add()s the state of the merge
    function equals the merge of n single-row runs of one key (sequence 0..n-1)."""

    def __init__(self, factory, row_type):
        self.schema = KeyValueSchema(RowType((DataField("_KEY_k", "INT", False),)), row_type)
        self.spec = factory.create()
        self.rows = []

    def reset(self):
        self.rows = []

    def add(self, *f, kind=RowKind.INSERT):
        self.rows.append((1, len(self.rows), int(kind)) + tuple(f))

    def validate(self, *f):
        assert len(self.rows) >= 2
        runs = [KeyValueBatch.from_rows(self.schema, [r]) for r in self.rows]
        got = assert_same(self.schema, self.spec, runs)
        assert got.n_rows == 1 and got.to_rows()[0][3:] == tuple(f)


def _int_row_type(n):
    return RowType(tuple(DataField(f"f{i}", "INT", True) for i in range(n)))


SEQ_GROUP_OPTS = {"fields.f3.sequence-group": "f1,f2", "fields.f6.sequence-group": "f4,f5"}
MULTI_SEQ_OPTS = {"fields.f3,f4.sequence-group": "f1,f2", "fields.f7,f8.sequence-group": "f5,f6"}
_D = RowKind.DELETE


def test_sequence_group_known_answers():
    """PartialUpdateMergeFunctionTest.java:64-97 (testSequenceGroup)."""
    rt = _int_row_type(7)
    d = GpuFuncDriver(PartialUpdateMergeFunction.factory(SEQ_GROUP_OPTS, rt, ["f0"]), rt)
    d.add(1, 1, 1, 1, 1, 1, 1)
    d.add(1, 2, 2, 2, 2, 2, None)
    d.validate(1, 2, 2, 2, 1, 1, 1)
    d.add(1, 3, 3, 1, 3, 3, 3)
    d.validate(1, 2, 2, 2, 3, 3, 3)
    d.add(1, 1, 1, 3, 1, 1, None, kind=_D)
    d.validate(1, None, None, 3, 3, 3, 3)
    d.add(1, 1, 1, 3, 1, 1, 4, kind=_D)
    d.validate(1, None, None, 3, None, None, 4)
    d.add(1, 4, 4, 4, 5, 5, 5)
    d.validate(1, 4, 4, 4, 5, 5, 5)
    d.add(1, 1, 1, 6, 1, 1, 6, kind=_D)
    d.validate(1, None, None, 6, None, None, 6)


def test_sequence_group_partial_delete_known_answers():
    """PartialUpdateMergeFunctionTest.java:99-134 ('partial-update.remove-record-on-sequence-group')."""
    rt = _int_row_type(7)
    opts = dict(SEQ_GROUP_OPTS, **{"partial-update.remove-record-on-sequence-group": "f6"})
    d = GpuFuncDriver(PartialUpdateMergeFunction.factory(opts, rt, ["f0"]), rt)
    d.add(1, 1, 1, 1, 1, 1, 1)
    d.add(1, 2, 2, 2, 2, 2, None)
    d.validate(1, 2, 2, 2, 1, 1, 1)
    d.add(1, 3, 3, 1, 3, 3, 3)
    d.validate(1, 2, 2, 2, 3, 3, 3)
    d.add(1, 1, 1, 3, 1, 1, None, kind=_D)
    d.validate(1, None, None, 3, 3, 3, 3)
    d.add(1, 1, 1, 3, 1, 1, 4, kind=_D)
    d.validate(1, 1, 1, 3, 1, 1, 4)
    d.add(1, 4, 4, 4, 5, 5, 5)
    d.validate(1, 4, 4, 4, 5, 5, 5)
    d.add(1, 1, 1, 6, 1, 1, 6, kind=_D)
    d.validate(1, 1, 1, 6, 1, 1, 6)


def test_multi_sequence_fields_known_answers():
    """PartialUpdateMergeFunctionTest.java:175-217 (two sequence fields per group)."""
    rt = _int_row_type(9)
    d = GpuFuncDriver(PartialUpdateMergeFunction.factory(MULTI_SEQ_OPTS, rt, ["f0"]), rt)
    d.add(1, None, None, None, None, 1, 1, 1, 3)
    d.add(1, 2, 2, None, None, 2, 2, 1, 3)
    d.validate(1, None, None, None, None, 2, 2, 1, 3)
    d.reset()
    d.add(1, 1, 1, 1, 1, 1, 1, 1, 3)
    d.add(1, 2, 2, 2, 2, 2, 1, 1, None)
    d.validate(1, 2, 2, 2, 2, 1, 1, 1, 3)
    d.add(1, 1, 3, 1, 3, 3, 3, 3, 2)
    d.validate(1, 2, 2, 2, 2, 3, 3, 3, 2)
    d.add(1, 1, 1, 3, 3, 1, 1, None, None, kind=_D)
    d.validate(1, None, None, 3, 3, 3, 3, 3, 2)
    d.add(1, 1, 1, 3, 1, 1, 1, 4, 4, kind=_D)
    d.validate(1, None, None, 3, 3, None, None, 4, 4)
    d.add(1, 4, 4, 4, 4, 5, 5, 5, 5)
    d.validate(1, 4, 4, 4, 4, 5, 5, 5, 5)
    d.add(1, 1, 1, 6, 1, 1, 1, 6, 1, kind=_D)
    d.validate(1, None, None, 6, 1, None, None, 6, 1)


def _seq_group_schema():
    vt = RowType((DataField("pk", "BIGINT", False),
                  DataField("a", "BIGINT", True), DataField("b", "VARCHAR(24)", True), DataField("g1", "INT", True),
                  DataField("c", "DOUBLE", True), DataField("d", "INT", True),
                  DataField("g2a", "INT", True), DataField("g2b", "BIGINT", True),
                  DataField("e", "BIGINT", True), DataField("s", "VARCHAR(24)", True)))
    return KeyValueSchema.of(vt, ["pk"])


def _coarsen_sequence_fields(schema, runs, names, modulo):
    """Small value ranges for the sequence fields so that ties and reversals between runs are common."""
    idx = [schema.n_key + 2 + [f.name for f in schema.value_type.fields].index(nm) for nm in names]
    for run in runs:
        for ci in idx:
            col = run.columns[ci]
            col.data = (np.abs(col.data) % modulo).astype(col.data.dtype)
    return runs


@pytest.mark.parametrize("mode", ["inserts_only", "ignore_delete", "retract", "partial_delete"])
@pytest.mark.parametrize("n_runs,total", [(3, 4000), (16, 60000)])
def test_sequence_groups_match_oracle(mode, n_runs, total):
    """'fields.<seq>.sequence-group': a group's fields follow the record with the greatest group sequence
    (PartialUpdateMergeFunction.java:190-247); retracts with sequence groups (:271-342)."""
    schema = _seq_group_schema()
    opts = {"fields.g1.sequence-group": "a,b", "fields.g2a,g2b.sequence-group": "c,d"}
    if mode == "ignore_delete":
        opts["ignore-delete"] = "true"
    if mode == "partial_delete":
        opts["partial-update.remove-record-on-sequence-group"] = "g2a,g2b"
    runs = datagen.make_runs(schema, n_runs, total, seed=21, null_prob=0.3,
                             delete_prob=0.0 if mode == "inserts_only" else 0.15)
    runs = _coarsen_sequence_fields(schema, runs, ["g1", "g2a", "g2b"], 3)
    spec = PartialUpdateMergeFunction.factory(opts, schema.value_type, ["pk"]).create()
    assert_same(schema, spec, runs)
    assert_same(schema, spec.with_drop_delete(), runs)


def test_sequence_group_specs_the_device_refuses():
    vt = RowType((DataField("f0", "INT", True), DataField("f1", "INT", True), DataField("f2", "STRING", True)))
    schema = KeyValueSchema(RowType((DataField("_KEY_k", "INT", False),)), vt)
    run = KeyValueBatch.from_rows(schema, [(1, 0, 0, 1, 1, "a")])
    # an aggregate function on a var-len field inside a sequence group
    spec = PartialUpdateMergeFunction.factory({"fields.f1.sequence-group": "f2",
                                               "fields.f2.aggregate-function": "last_value"}, vt, ["f0"]).create()
    with pytest.raises(N.UnsupportedOnDevice):
        merge_runs(schema, spec, [run])


def test_sequence_group_aggregates_known_answers():
    """Aggregate functions inside sequence groups (PartialUpdateMergeFunction.java:228-244, 323-339):
    PartialUpdateMergeFunctionTest.java:219-275 (default agg), :569-616 (first_value / last_value, in order and
    reversed), :618-742 (sum / last_value / last_non_null_value with retracts and ignore-retract)."""
    rt = _int_row_type(7)
    opts = dict(SEQ_GROUP_OPTS, **{"fields.default-aggregate-function": "last_non_null_value"})
    d = GpuFuncDriver(PartialUpdateMergeFunction.factory(opts, rt, ["f0"]), rt)
    d.add(1, 1, 1, 1, 1, 1, 1)
    d.add(1, 2, 2, 2, 2, 2, None)
    d.validate(1, 2, 2, 2, 1, 1, 1)
    d.add(1, 3, 3, 1, 3, 3, 3)
    d.validate(1, 2, 2, 2, 3, 3, 3)
    d.add(1, 4, None, 4, 5, None, 5)
    d.validate(1, 4, 2, 4, 5, 3, 5)

    rt = _int_row_type(9)
    opts = dict(MULTI_SEQ_OPTS, **{"fields.default-aggregate-function": "last_non_null_value"})
    d = GpuFuncDriver(PartialUpdateMergeFunction.factory(opts, rt, ["f0"]), rt)
    d.add(1, 1, 1, 1, 1, 1, 1, 1, 1)
    d.add(1, 2, 2, 2, 2, 2, 2, None, None)
    d.validate(1, 2, 2, 2, 2, 1, 1, 1, 1)
    d.add(1, 3, 3, 1, 1, 3, 3, 3, 3)
    d.validate(1, 2, 2, 2, 2, 3, 3, 3, 3)
    d.add(1, 4, None, 4, 4, 5, None, 5, 5)
    d.validate(1, 4, 2, 4, 4, 5, 3, 5, 5)

    rt = _int_row_type(4)
    opts = {"fields.f1.sequence-group": "f2,f3", "fields.f2.aggregate-function": "first_value",
            "fields.f3.aggregate-function": "last_value"}
    d = GpuFuncDriver(PartialUpdateMergeFunction.factory(opts, rt, ["f0"]), rt)
    d.add(1, 1, 1, 1)
    d.add(1, 2, 2, 2)
    d.validate(1, 2, 1, 2)
    d.add(1, 0, 3, 3)
    d.validate(1, 2, 3, 2)

    rt = _int_row_type(5)
    opts = {"fields.f1,f2.sequence-group": "f3,f4", "fields.f3.aggregate-function": "first_value",
            "fields.f4.aggregate-function": "last_value"}
    d = GpuFuncDriver(PartialUpdateMergeFunction.factory(opts, rt, ["f0"]), rt)
    d.add(1, 1, 1, 1, 1)
    d.add(1, 2, 2, 2, 2)
    d.validate(1, 2, 2, 1, 2)
    d.add(1, 0, 1, 3, 3)
    d.validate(1, 2, 2, 3, 2)

    rt = _int_row_type(8)
    opts = {"fields.f1.sequence-group": "f2,f3,f4", "fields.f7.sequence-group": "f6",
            "fields.f0.aggregate-function": "listagg", "fields.f2.aggregate-function": "sum",
            "fields.f4.aggregate-function": "last_value", "fields.f6.aggregate-function": "last_non_null_value",
            "fields.f4.ignore-retract": "true", "fields.f6.ignore-retract": "true"}
    d = GpuFuncDriver(PartialUpdateMergeFunction.factory(opts, rt, ["f0"]), rt)
    d.add(1, 1, 1, 1, 1, 1, 1, 1)
    d.add(1, 2, 1, 2, 2, 2, 2, 0)
    d.validate(1, 2, 2, 2, 2, 2, 1, 1)
    d.add(1, 1, 1, 1, 1, 1, 2, 0)
    d.validate(1, 2, 3, 2, 2, 1, 1, 1)
    d.add(1, 1, -1, 1, 1, 2, 2, 0)
    d.add(1, 3, None, None, None, None, None, 2)
    d.validate(1, 3, 2, None, None, 2, 1, 2)
    d.add(1, 3, 1, 1, 1, 1, 1, 3)
    d.validate(1, 3, 3, 1, 1, 1, 1, 3)
    d.add(1, 3, 2, 1, 1, 1, 1, 3, kind=RowKind.UPDATE_BEFORE)
    d.validate(1, 3, 1, None, 1, 1, 1, 3)
    d.add(1, 3, 2, 1, 1, 1, 1, 3, kind=_D)
    d.validate(1, 3, -1, None, 1, 1, 1, 3)
    d.add(1, 2, 2, 1, 1, 1, 1, 3, kind=_D)
    d.validate(1, 3, -3, None, 1, 1, 1, 3)


@pytest.mark.parametrize("mode", ["inserts_only", "retract"])
def test_sequence_group_aggregates_match_oracle(mode):
    schema = _seq_group_schema()
    opts = {"fields.g1.sequence-group": "a,b", "fields.g2a,g2b.sequence-group": "c,d",
            "fields.a.aggregate-function": "sum", "fields.c.aggregate-function": "max",
            "fields.d.aggregate-function": "first_value"}
    if mode == "retract":
        opts.update({"fields.c.ignore-retract": "true", "fields.d.ignore-retract": "true"})
    for n_runs, total in ((3, 4000), (16, 60000)):
        runs = datagen.make_runs(schema, n_runs, total, seed=23, null_prob=0.3,
                                 delete_prob=0.15 if mode == "retract" else 0.0)
        runs = _coarsen_sequence_fields(schema, runs, ["g1", "g2a", "g2b"], 3)
        spec = PartialUpdateMergeFunction.factory(opts, schema.value_type, ["pk"]).create()
        assert_same(schema, spec, runs)


# ---------------------------------------------------------------- streaming in key ranges

@pytest.mark.parametrize("engine", ["deduplicate", "partial-update", "aggregate"])
@pytest.mark.parametrize("target_rows,depth", [(700, 3), (5000, 2), (10 ** 9, 1)])
def test_range_streaming_equals_single_batch(engine, target_rows, depth):
    """RangeStreamingMergeReader: the batches of the key ranges, concatenated, are the single merged batch
    (sub-runs start at 8-row boundaries + pg_merge_rebind start rows; var-len columns keep absolute offsets)."""
    from paimon_b200.merge_tree_readers import concat_batches
    from paimon_b200.sort_merge_reader import RangeStreamingMergeReader
    schema = datagen.schema_c3(n_i64=3, n_f64=2, n_str=2)
    runs = datagen.make_runs(schema, 5, 20000, seed=31, null_prob=0.4, delete_prob=0.1 if engine == "deduplicate" else 0.0)
    runs.append(datagen.make_runs(schema, 1, 40, seed=77, null_prob=0.4)[0])        # a tiny run: empty sub-runs
    if engine == "deduplicate":
        spec = DeduplicateMergeFunction.factory().create()
    elif engine == "partial-update":
        spec = PartialUpdateMergeFunction.factory({}, schema.value_type, ["pk"]).create()
    else:
        spec = AggregateMergeFunction.factory({"fields.d0.aggregate-function": "sum",
                                               "fields.i1.aggregate-function": "max"}, schema.value_type, ["pk"]).create()
    want = pyoracle.merge(schema, spec, runs, pyoracle.SORT_LOSER_TREE)
    rd = RangeStreamingMergeReader(schema, runs, spec, target_rows=target_rows, depth=depth)
    try:
        batches = []
        while True:
            b = rd.read_batch()
            if b is None:
                break
            batches.append(b)
    finally:
        rd.close()
    if target_rows < 10000:
        assert len(batches) > 3
    got = concat_batches(schema, batches)
    assert got.equals(want), got.first_difference(want)
    for a, b in zip(batches, batches[1:]):          # key-disjoint and ascending
        assert a.columns[0].data[a.n_rows - 1] < b.columns[0].data[0]


def test_device_matches_golden_file():
    """The committed golden vectors (reference test inputs + the reference calculators' results), through the C ABI."""
    from golden_util import load_cases, records, spec_for
    from reusing_test_data import from_batch
    n = 0
    for case in load_cases():
        runs = [to_batch(records(r)) for r in case["readers"]]
        for name, want in case["expected"].items():
            got = merge_runs(SCHEMA, spec_for(name), runs)
            assert from_batch(got) == records(want), (case["name"], name)
            n += 1
    assert n >= 100


def test_arrow_c_data_export_matches_fetch():
    """pg_export_arrow: the merged batch through the Arrow C Data Interface, imported by pyarrow the way the JVM
    imports it (Data.importVectorSchemaRoot -> ArrowBatchReader, which maps columns by the Paimon field names);
    whole batch and row ranges that do not start at byte boundaries of the validity bitmaps."""
    import pyarrow as pa
    from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader, export_arrow
    from parquet_util import arrow_to_batch
    rng = random.Random(23)
    schema, runs = random_all_types_runs(rng, 5, 400, 700, [0, 0, 2, 3])
    spec = DeduplicateMergeFunction.factory().create()
    rd = SortMergeReader.create_sort_merge_reader([SortedRunReader(schema, b) for b in runs], None, None, spec)
    try:
        rd.execute()
        want = rd.fetch()
        n = want.n_rows
        full = export_arrow(schema, rd._merge_h)
        assert full.schema.names == [f.name for f in schema.file_fields()]
        assert full.schema.names[schema.n_key] == "_SEQUENCE_NUMBER" and full.schema.names[schema.n_key + 1] == "_VALUE_KIND"
        got = arrow_to_batch(schema, pa.Table.from_batches([full]))
        assert got.equals(want), got.first_difference(want)
        from paimon_b200.sort_merge_reader import slice_rows
        for lo, hi in ((0, 1), (3, 77), (129, n), (n - 1, n), (5, 5)):
            part = export_arrow(schema, rd._merge_h, lo, hi - lo)
            assert part.num_rows == hi - lo
            if hi > lo:
                g = arrow_to_batch(schema, pa.Table.from_batches([part]))
                w = slice_rows(want, lo, hi)
                assert g.equals(w), (lo, hi, g.first_difference(w))
        del full, part
    finally:
        rd.close()
