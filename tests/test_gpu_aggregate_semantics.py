"""The device's aggregate functions against the independent reference (tests/agg_reference.py), keyed by LOGICAL type,
at the type's edge values; and against the C oracle row for row.  Needs an H100.

Float rule: sum / product results are compared bit for bit except that all NaNs count as equal (Java does not fix the
payload of a NaN an add or multiply returns, and neither does the GPU); max / min / first / last select an input and
are compared bit for bit, NaN payload included."""
import random
import zlib
from decimal import Decimal

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import agg_reference as R
from oracle import pyoracle
from paimon_b200 import _native as N
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.merge_function import AggregateMergeFunction, PartialUpdateMergeFunction
from paimon_b200.sort_merge_reader import merge_runs
from paimon_b200.types import DataField, KeyValueSchema, RowType

from test_agg_semantics_cpu import AGGS_OF, Fold, cell, check_against_reference, ref_cell, same_value

pytestmark = pytest.mark.gpu


def assert_same_as_oracle(schema, spec, runs, got, arith_cols=()):
    """Every cell of the device batch against the oracle's; value columns in `arith_cols` (value-field indexes) are
    sum / product results, where any NaN equals any NaN."""
    want = pyoracle.merge(schema, spec, runs)
    assert got.n_rows == want.n_rows
    nk = schema.n_key + 2
    for ci, (g, w) in enumerate(zip(got.columns, want.columns)):
        agg = "sum" if ci >= nk and (ci - nk) in arith_cols else "select"
        for i in range(got.n_rows):
            a, b = cell(g, i), cell(w, i)
            assert same_value(agg, a, b), f"column {ci} row {i}: {a!r} != {b!r}"


CASES = [(t, a) for t, aggs in AGGS_OF.items() for a in aggs]


@pytest.mark.parametrize("logical,agg", CASES)
@pytest.mark.parametrize("mode", ["retract", "ignore_retract"])
def test_edge_matrix(logical, agg, mode):
    """~2,000 keys, 1 to 32 records each spread over 32 runs (one record per run: the longest fold a key can have),
    values drawn from the type's edges, retracts included."""
    fold = Fold(logical, agg, mode == "ignore_retract", n_keys=2000, max_records=32, n_runs=32,
                seed=zlib.crc32(f"gpu/{logical}/{agg}/{mode}".encode()))
    got = merge_runs(fold.schema, fold.spec, fold.runs)
    check_against_reference(fold, got)
    assert_same_as_oracle(fold.schema, fold.spec, fold.runs, got, arith_cols=(1,) if agg in ("sum", "product") else ())


@pytest.mark.parametrize("logical,agg", [("DECIMAL(18,4)", "sum"), ("DECIMAL(9,2)", "product"),
                                         ("DECIMAL(10,0)", "product"), ("FLOAT", "sum"), ("DOUBLE", "max"),
                                         ("BIGINT", "product"), ("STRING", "min")])
def test_multi_tile(logical, agg):
    """The same generator at ~200k rows over 16 runs: folds in every plan tile and partition level."""
    fold = Fold(logical, agg, False, n_keys=24000, max_records=16, n_runs=16, seed=11)
    assert sum(r.n_rows for r in fold.runs) > 150_000
    got = merge_runs(fold.schema, fold.spec, fold.runs)
    check_against_reference(fold, got)
    assert_same_as_oracle(fold.schema, fold.spec, fold.runs, got, arith_cols=(1,) if agg in ("sum", "product") else ())


# ---------------------------------------------------------------------------------------------- sequence groups

PU_FIELDS = [("k", "INT"), ("g1", "BIGINT"), ("a", "DECIMAL(18,4)"), ("b", "FLOAT"), ("c", "DECIMAL(9,2)"),
             ("g2", "BIGINT"), ("d", "FLOAT"), ("e", "DECIMAL(10,0)"), ("f", "DECIMAL(15,2)")]
PU_OPTIONS = {"fields.g1.sequence-group": "a,b,c", "fields.g2.sequence-group": "d,e,f",
              "fields.a.aggregate-function": "sum", "fields.b.aggregate-function": "product",
              "fields.c.aggregate-function": "max", "fields.d.aggregate-function": "sum",
              "fields.e.aggregate-function": "product", "fields.f.aggregate-function": "product"}


@pytest.mark.parametrize("retracts", [False, True])
def test_partial_update_sequence_groups(retracts):
    """sum / product / max on DECIMAL and FLOAT fields inside sequence groups (the agg_pair path): a record whose
    group sequence is older than the accumulated one folds reversed (aggReversed); a NULL group sequence skips it."""
    from test_agg_semantics_cpu import edge_values
    vt = RowType(tuple(DataField(n, t, n != "k") for n, t in PU_FIELDS))
    schema = KeyValueSchema.of(vt, ["k"])
    spec = PartialUpdateMergeFunction.factory(PU_OPTIONS, vt, ["k"]).create()
    ref = R.PartialUpdateReference(PU_FIELDS, ["k"], PU_OPTIONS)
    rng = random.Random(21 + retracts)
    edges = {n: edge_values(t) for n, t in PU_FIELDS if n not in ("k", "g1", "g2")}
    n_runs = 16
    rows_of_run = [[] for _ in range(n_runs)]
    expected = {}
    for key in range(3000):
        n = rng.randint(1, n_runs)
        records = []
        for _ in range(n):
            row = [key, None if rng.random() < 0.15 else rng.randrange(0, 6)]
            row += [None if rng.random() < 0.1 else rng.choice(edges[f]) for f in ("a", "b", "c")]
            row += [None if rng.random() < 0.15 else rng.randrange(0, 6)]
            row += [None if rng.random() < 0.1 else rng.choice(edges[f]) for f in ("d", "e", "f")]
            kind = rng.choice([R.INSERT, R.INSERT, R.UPDATE_BEFORE]) if retracts else R.INSERT
            records.append((kind, row))
        try:
            expected[key] = ref.merge(records)
        except R.JavaException:
            records = [(R.INSERT, r) for _, r in records]
            expected[key] = ref.merge(records)
        for j, (r, (kind, row)) in enumerate(zip(sorted(rng.sample(range(n_runs), n)), records)):
            rows_of_run[r].append((key, j, kind, *row))
    runs = [KeyValueBatch.from_rows(schema, rows) for rows in rows_of_run if rows]
    got = merge_runs(schema, spec, runs)
    keys = [int(k) for k in got.key_column(0).data[: got.n_rows]]
    assert keys == sorted(expected)
    arith = {"a", "b", "d", "e", "f"}
    bad = []
    for vi, (name, logical) in enumerate(PU_FIELDS):
        col = got.value_column(vi)
        for i, k in enumerate(keys):
            g, w = cell(col, i), ref_cell(logical, expected[k][1][vi])
            if not same_value("sum" if name in arith else "select", g, w):
                bad.append((name, k, g, w))
    assert not bad, f"{len(bad)} cells differ, first: {bad[:4]}"
    assert [int(x) for x in got.value_kinds] == [expected[k][0] for k in keys]
    assert_same_as_oracle(schema, spec, runs, got, arith_cols=(2, 3, 6, 7, 8))


# ---------------------------------------------------------------------------------------------- error paths

def _two_records(logical, acc, inp):
    vt = RowType((DataField("k", "INT", False), DataField("v", logical, True)))
    schema = KeyValueSchema.of(vt, ["k"])
    spec = AggregateMergeFunction.factory({"fields.v.aggregate-function": "product"}, vt, ["k"]).create()
    # other keys around the failing one, so that the error is raised from inside a full tile
    runs = [KeyValueBatch.from_rows(schema, [(k, 0, R.INSERT, k, acc if k == 500 else 3) for k in range(1000)]),
            KeyValueBatch.from_rows(schema, [(k, 1, R.UPDATE_BEFORE if k == 500 else R.INSERT, k,
                                              inp if k == 500 else 2) for k in range(1000)])]
    return schema, spec, runs


@pytest.mark.parametrize("logical,acc,inp,msg", [
    ("INT", 7, 0, "/ by zero"),
    ("BIGINT", 7, 0, "/ by zero"),
    ("DECIMAL(15,2)", 100, 300, "Non-terminating decimal expansion; no exact representable decimal result."),
    ("DECIMAL(9,2)", 100, 0, "Division by zero"),
    ("DECIMAL(18,4)", 0, 0, "Division undefined"),
])
def test_retract_divide_errors(logical, acc, inp, msg):
    with pytest.raises(R.JavaException, match=msg[:20]):
        R.FieldAgg("product", logical).retract(acc, inp)
    schema, spec, runs = _two_records(logical, acc, inp)
    with pytest.raises(N.MergeFunctionError, match=msg[:20]):
        merge_runs(schema, spec, runs)
    with pytest.raises(pyoracle.OracleError, match=msg[:20]):
        pyoracle.merge(schema, spec, runs)


def test_decimal_over_18_digits_is_refused_by_the_library():
    """pg_merge_spec_create refuses DECIMAL(p > 18) even when a caller bypasses the Python type mapping."""
    vt = RowType((DataField("k", "INT", False), DataField("v", "DECIMAL(18,2)", True)))
    schema = KeyValueSchema.of(vt, ["k"])
    spec = AggregateMergeFunction.factory({"fields.v.aggregate-function": "sum"}, vt, ["k"]).create()
    spec.decimal = [0, 38 << 8 | 2]
    runs = [KeyValueBatch.from_rows(schema, [(1, 0, R.INSERT, 1, 5)])]
    with pytest.raises(N.UnsupportedOnDevice, match="DECIMAL"):
        merge_runs(schema, spec, runs)


# ---------------------------------------------------------------------------------------------- decode -> aggregate

DEC_FIELDS = [("k", "INT"), ("p5", "DECIMAL(5,2)"), ("p9", "DECIMAL(9,2)"), ("p18", "DECIMAL(18,4)"),
              ("p10", "DECIMAL(10,0)")]
DEC_AGGS = {"p5": "sum", "p9": "product", "p18": "sum", "p10": "max"}


def _write_decimal_file(path, rows, encoding):
    """A data file as Paimon stores decimals: DECIMAL(p <= 9) as INT32, p <= 18 as INT64 (unscaled)."""
    cols = {"_KEY_k": pa.array([r[0] for r in rows], pa.int32()),
            "_SEQUENCE_NUMBER": pa.array([r[1] for r in rows], pa.int64()),
            "_VALUE_KIND": pa.array([r[2] for r in rows], pa.int8()),
            "k": pa.array([r[3] for r in rows], pa.int32())}
    for vi, (name, logical) in enumerate(DEC_FIELDS[1:], start=4):
        p, s = R.decimal_ps(logical)
        vals = [None if r[vi] is None else Decimal(r[vi]).scaleb(-s) for r in rows]
        cols[name] = pa.array(vals, pa.decimal128(p, s))
    table = pa.table(cols)
    kw = dict(compression="none", data_page_version="1.0", write_statistics=False, store_decimal_as_integer=True,
              data_page_size=4096)
    if encoding == "dictionary":
        kw["use_dictionary"] = True
    else:
        kw["use_dictionary"] = False
        kw["column_encoding"] = {n: encoding for n in table.column_names if n not in ("_VALUE_KIND",)}
    pq.write_table(table, path, **kw)
    meta = pq.ParquetFile(path).schema.to_arrow_schema()
    return table, meta


@pytest.mark.parametrize("encoding", ["PLAIN", "dictionary", "DELTA_BINARY_PACKED"])
def test_decode_then_aggregate_decimals(tmp_path, encoding):
    from paimon_b200.format import read_section
    from paimon_b200.merge_tree_readers import DataFileMeta, MergeFileSplitRead, concat_batches
    from test_agg_semantics_cpu import decimal_edges
    vt = RowType(tuple(DataField(n, t, n != "k") for n, t in DEC_FIELDS))
    schema = KeyValueSchema.of(vt, ["k"])
    opts = {f"fields.{n}.aggregate-function": a for n, a in DEC_AGGS.items()}
    rng = random.Random(5)
    edges = {n: decimal_edges(*R.decimal_ps(t)) for n, t in DEC_FIELDS[1:]}
    ref = R.AggregateReference(DEC_FIELDS, ["k"], opts)
    n_files, records_of = 6, {}
    paths, metas = [], []
    for f in range(n_files):
        rows = []
        for k in range(0, 3000, 1 + f % 3):
            vals = [None if rng.random() < 0.15 else rng.choice(edges[n]) for n, _ in DEC_FIELDS[1:]]
            rows.append((k, f, R.INSERT, k, *vals))
            records_of.setdefault(k, []).append((R.INSERT, [k] + vals))
        path = str(tmp_path / f"dec-{f}.parquet")
        table, arrow_schema = _write_decimal_file(path, rows, encoding)
        assert str(arrow_schema.field("p9").type) == "decimal128(9, 2)"
        pf = pq.ParquetFile(path)
        phys = {pf.schema.column(i).name: pf.schema.column(i).physical_type for i in range(len(pf.schema))}
        assert phys["p5"] == "INT32" and phys["p9"] == "INT32" and phys["p18"] == "INT64" and phys["p10"] == "INT64"
        # decode alone: every value column against pyarrow's unscaled values (INT32 pages widened to INT64)
        readers, _ = read_section(schema, [(open(path, "rb").read(), 0)], 1)
        try:
            got = readers[0].read_batch()
        finally:
            for r in readers:
                r.close()
        for vi, (name, logical) in enumerate(DEC_FIELDS[1:], start=1):
            s = R.decimal_ps(logical)[1]
            want = [None if v is None else int(v.scaleb(s)) for v in table.column(name).to_pylist()]
            assert got.value_column(vi).to_pylist() == want, f"{encoding} file {f} column {name}"
        paths.append(path)
        metas.append(DataFileMeta(path, 0, len(rows), rows[0][0], rows[-1][0], level=0))
    # decode -> merge through MergeFileSplitRead, against the reference
    spec_f = AggregateMergeFunction.factory(opts, vt, ["k"])
    rd = MergeFileSplitRead(schema, spec_f).create_merge_reader(metas)
    batches = []
    while True:
        b = rd.read_batch()
        if b is None:
            break
        batches.append(b)
    rd.close()
    got = concat_batches(schema, batches)
    keys = [int(x) for x in got.key_column(0).data[: got.n_rows]]
    assert keys == sorted(records_of)
    for vi, (name, logical) in enumerate(DEC_FIELDS[1:], start=1):
        col = got.value_column(vi).to_pylist()
        want = [ref.merge(records_of[k])[1][vi] for k in keys]
        assert col == want, f"{encoding}: column {name}"
