"""tests/bench_shapes.py against bench.py, without importing bench.py: its syntax tree is read with ast.  The restated
constants and WORKLOADS entries must equal the bench's values, the schema and bucket functions must have the bench's
syntax trees, and c5_writer_args must be the keyword arguments of the bench's pyarrow write_table call for both
codecs.  When the benchmark's shapes move, this fails until the tests' copy follows."""
import ast
import inspect
import os

import pytest

import bench_shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bench_tree(path=os.path.join(ROOT, "bench.py")):
    with open(path) as f:
        return ast.parse(f.read())


def assignment(tree, name):
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == name for t in node.targets):
            return node.value
    raise KeyError(name)


def function(tree, name):
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == name:
            return node
    raise KeyError(name)


def constant(node, **names):
    """The value of a constant expression (literals, arithmetic, shifts, dict(...) of them) with `names` bound."""
    return eval(compile(ast.Expression(node), "<bench.py>", "eval"), {"__builtins__": {"dict": dict}}, names)


def test_page_and_row_group_rows():
    tree = bench_tree()
    assert constant(assignment(tree, "PARQUET_PAGE_ROWS")) == bench_shapes.PARQUET_PAGE_ROWS
    assert constant(assignment(tree, "PARQUET_GROUP_ROWS")) == bench_shapes.PARQUET_GROUP_ROWS


@pytest.mark.parametrize("workload", sorted(bench_shapes.WORKLOADS))
def test_workload_entries(workload):
    workloads = constant(assignment(bench_tree(), "WORKLOADS"))
    assert workloads[workload] == bench_shapes.WORKLOADS[workload]


@pytest.mark.parametrize("name", ["schema_c4", "schema_c5", "c5_bucket"])
def test_functions_have_the_bench_syntax_tree(name):
    ours = ast.parse(inspect.getsource(getattr(bench_shapes, name))).body[0]
    assert ast.dump(ours) == ast.dump(function(bench_tree(), name))


@pytest.mark.parametrize("name", ["_splitmix64", "_hex_keys", "gen_device_run"])
def test_device_generator_has_the_bench_syntax_tree(name):
    """tests/device_runs.py restates the generator of the bench's C2, C3 and C4 inputs."""
    import device_runs
    ours = ast.parse(inspect.getsource(getattr(device_runs, name))).body[0]
    assert ast.dump(ours) == ast.dump(function(bench_tree(), name))


def test_an_edited_generator_is_noticed(tmp_path):
    """A bench.py whose generator draws string lengths from another range no longer matches the restatement."""
    import device_runs
    with open(os.path.join(ROOT, "bench.py")) as f:
        src = f.read()
    assert "lens = 8 + ((h >> 3) & 0xffff) % 17" in src
    moved = tmp_path / "bench.py"
    moved.write_text(src.replace("lens = 8 + ((h >> 3) & 0xffff) % 17", "lens = 8 + ((h >> 3) & 0xffff) % 16", 1))
    ours = ast.parse(inspect.getsource(device_runs.gen_device_run)).body[0]
    assert ast.dump(ours) != ast.dump(function(bench_tree(str(moved)), "gen_device_run"))


@pytest.mark.parametrize("codec", ["none", "zstd"])
def test_c5_writer_arguments(codec):
    calls = [n for n in ast.walk(function(bench_tree(), "c5_bucket"))
             if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr == "write_table"]
    assert len(calls) == 1
    kwargs = {}
    for kw in calls[0].keywords:
        value = constant(kw.value, codec=codec)
        if kw.arg is None:                                         # **{...}
            kwargs.update(value)
        else:
            kwargs[kw.arg] = value
    assert kwargs == bench_shapes.c5_writer_args(codec)
    assert kwargs["data_page_version"] == "1.0" and kwargs["use_dictionary"]


def test_schemas_as_objects():
    c4, c5 = bench_shapes.schema_c4(), bench_shapes.schema_c5()
    assert [(f.name, f.type, f.nullable) for f in c4.file_fields()][3:] == \
        [("pk", "VARCHAR(16)", False)] + [(f"i{i}", "BIGINT", True) for i in range(4)] + \
        [(f"d{i}", "DOUBLE", True) for i in range(2)] + [(f"n{i}", "INT", True) for i in range(2)] + \
        [(f"s{i}", "VARCHAR(64)", True) for i in range(3)]
    assert c5.n_key == 2 and c5.n_cols == 20


@pytest.mark.parametrize("nulls", [0.0, 0.4, 1.0])
@pytest.mark.parametrize("sliced", [False, True])
def test_arrow_to_column_equals_the_python_value_path(nulls, sliced):
    """The buffer path of parquet_util.arrow_to_column, which the bench-shape tests use on millions of rows, builds
    the same buffers as Column.from_pylist over the arrow values: every type it takes, NULLs, sliced arrays, and
    string payload left under NULL slots."""
    import numpy as np
    import pyarrow as pa

    from paimon_b200.columnar import Column
    from paimon_b200.types import PhysicalType
    from parquet_util import arrow_to_column

    rng = np.random.default_rng(int(nulls * 10) + sliced)
    n = 1000
    mask = rng.random(n) < nulls
    words = [bytes(rng.integers(0, 256, rng.integers(0, 20), dtype=np.uint8)) for _ in range(n)]
    cases = [(PhysicalType.INT8, pa.array(rng.integers(-128, 128, n).astype(np.int8), mask=mask)),
             (PhysicalType.INT32, pa.array(rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32), mask=mask)),
             (PhysicalType.INT64, pa.array(rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64), mask=mask)),
             (PhysicalType.INT64, pa.array(rng.integers(0, 100, n).astype(np.int32), mask=mask)),      # widened
             (PhysicalType.FLOAT, pa.array(rng.standard_normal(n).astype(np.float32), mask=mask)),
             (PhysicalType.DOUBLE, pa.array(np.where(rng.random(n) < 0.1, -0.0, rng.standard_normal(n)), mask=mask)),
             (PhysicalType.BOOL, pa.array(rng.random(n) < 0.5, mask=mask)),
             (PhysicalType.STRING, pa.array([w.hex() for w in words], pa.string(), mask=mask)),
             (PhysicalType.BINARY, pa.array(words, pa.binary(), mask=mask)),
             # payload under NULL slots, as a writer may leave it
             (PhysicalType.BINARY, pa.Array.from_buffers(pa.binary(), n, [pa.array(~mask).buffers()[1]] +
                                                         pa.array(words, pa.binary()).buffers()[1:], null_count=-1))]
    for t, arr in cases:
        if sliced:
            arr = arr.slice(13, n - 40)
        fast, slow = arrow_to_column(t, arr), Column.from_pylist(t, arr.to_pylist())
        assert fast.equals(slow), (t, arr.type)
        assert (fast.valid is None) == (slow.valid is None)
        assert fast.data.dtype == slow.data.dtype and fast.data.tobytes() == slow.data.tobytes(), (t, arr.type)
        assert (fast.offsets is None) == (slow.offsets is None)
        if fast.offsets is not None:
            assert fast.offsets.dtype == slow.offsets.dtype and np.array_equal(fast.offsets, slow.offsets)


def test_a_moved_constant_is_noticed(tmp_path):
    """The checks above read whatever bench.py says: a copy with another page-row limit no longer matches."""
    with open(os.path.join(ROOT, "bench.py")) as f:
        src = f.read()
    assert "PARQUET_PAGE_ROWS = 20_000" in src
    moved = tmp_path / "bench.py"
    moved.write_text(src.replace("PARQUET_PAGE_ROWS = 20_000", "PARQUET_PAGE_ROWS = 16_000", 1))
    assert constant(assignment(bench_tree(str(moved)), "PARQUET_PAGE_ROWS")) != bench_shapes.PARQUET_PAGE_ROWS
