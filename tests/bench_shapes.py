"""The inputs of bench.py's C3, C4 and C5 arms, restated for the tests so that they can be built at the benchmark's own
sizes without importing bench.py (which sets process-wide allocator settings when it is imported).

tests/test_bench_shapes_cpu.py holds every definition here to bench.py's: the constants and WORKLOADS entries by value,
the functions by their syntax trees.  If the benchmark's shapes move, that test fails until this file follows."""
import numpy as np

WORKLOADS = {
    "c3": dict(n_runs=16, rows=40_000_000, engine="partial-update", null_prob=0.5,
               desc="16-run partial-update, 50-col wide row (pk+20 i64+15 f64+14 varchar), 40M rows"),
    "c4": dict(n_runs=32, rows=16_000_000, engine="deduplicate", null_prob=0.5, delete_prob=0.05, drop_delete=True,
               desc="one bucket of a full compaction rewrite: 32 runs x 500K rows, varchar(16) pk + 4 i64 + 2 f64 + "
                    "2 i32 + 3 varchar, 5% deletes, drop-delete, output re-encoded to Parquet"),
}
PARQUET_PAGE_ROWS = 20_000          # parquet-mr's page row limit (RowDataParquetBuilder.java:63-99 pulls the defaults)
PARQUET_GROUP_ROWS = 400_000        # ~128 MiB row groups at c3's ~310 encoded bytes per row


def schema_c4():
    from paimon_b200.types import DataField, KeyValueSchema, RowType
    fields = [DataField("pk", "VARCHAR(16)", False)]
    fields += [DataField(f"i{i}", "BIGINT", True) for i in range(4)]
    fields += [DataField(f"d{i}", "DOUBLE", True) for i in range(2)]
    fields += [DataField(f"n{i}", "INT", True) for i in range(2)]
    fields += [DataField(f"s{i}", "VARCHAR(64)", True) for i in range(3)]
    return KeyValueSchema.of(RowType(tuple(fields)), ["pk"])


def schema_c5():
    """SURVEY §8d C5: pk (l_orderkey BIGINT, l_linenumber INT), 16 columns."""
    from paimon_b200.types import DataField, KeyValueSchema, RowType
    fields = [DataField("l_orderkey", "BIGINT", False), DataField("l_linenumber", "INT", False),
              DataField("l_partkey", "BIGINT", True), DataField("l_suppkey", "BIGINT", True),
              DataField("l_quantity", "DECIMAL(15,2)", True), DataField("l_extendedprice", "DECIMAL(15,2)", True),
              DataField("l_discount", "DECIMAL(15,2)", True), DataField("l_tax", "DECIMAL(15,2)", True),
              DataField("l_returnflag", "CHAR(1)", True), DataField("l_linestatus", "CHAR(1)", True),
              DataField("l_shipdate", "DATE", True), DataField("l_commitdate", "DATE", True),
              DataField("l_receiptdate", "DATE", True), DataField("l_shipinstruct", "CHAR(25)", True),
              DataField("l_shipmode", "CHAR(10)", True), DataField("l_comment", "VARCHAR(44)", True)]
    return KeyValueSchema.of(RowType(tuple(fields)), ["l_orderkey", "l_linenumber"])


def c5_bucket(schema, codec, seed=5):
    """One C5 bucket as parquet-mr-style files written by pyarrow on the host (dictionary on with parquet-mr's 1 MiB
    dictionary page limit, data page V1, ~128 MiB row groups; DECIMAL(15,2) / DATE in their physical INT64 / INT32
    form): 1 base run (83.3 %) + 4 update runs whose keys are resampled from the base.  parquet-mr closes a page at
    1 MiB OR 20 000 rows (parquet.page.row.count.limit, RowDataParquetBuilder.java:63-99 keeps the defaults), pyarrow
    only knows a byte limit: 160 KiB pages give the 20 000-row pages an 8-byte column gets from parquet-mr.
    Returns ([(file bytes, run)], rows in, expected columns)."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    rng = np.random.default_rng(seed)
    total = 1_000_000_000 // 64
    n_base = int(total * 5 / 6)
    n_upd = (total - n_base) // 4
    names = [f.name for f in schema.file_fields()]
    flags = [np.array([b"A", b"N", b"R"]), np.array([b"F", b"O"])]
    instr = np.array([b"DELIVER IN PERSON", b"COLLECT COD", b"NONE", b"TAKE BACK RETURN"])
    modes = np.array([b"REG AIR", b"AIR", b"RAIL", b"SHIP", b"TRUCK", b"MAIL", b"FOB"])

    def run_table(idx, seq0):
        n = len(idx)
        ok_, ln_ = pa.array(idx // 4), pa.array((idx % 4 + 1).astype(np.int32))
        # (a Paimon value row carries the primary-key fields too: _KEY_* copies + the table's own columns)
        cols = [ok_, ln_, pa.array(seq0 + np.arange(n, dtype=np.int64)), pa.array(np.zeros(n, np.int8)), ok_, ln_]
        part = rng.integers(1, 20_000_000, n)
        cols += [pa.array(part), pa.array(rng.integers(1, 1_000_000, n))]
        cols += [pa.array(rng.integers(100, 5_000_000, n)) for _ in range(4)]
        cols += [pa.array(flags[0][rng.integers(0, 3, n)]).cast(pa.string()), pa.array(flags[1][rng.integers(0, 2, n)]).cast(pa.string())]
        ship = rng.integers(8000, 10600, n).astype(np.int32)
        cols += [pa.array(ship), pa.array(ship + 30), pa.array(ship + 45)]
        cols += [pa.array(instr[rng.integers(0, 4, n)]).cast(pa.string()), pa.array(modes[rng.integers(0, 7, n)]).cast(pa.string())]
        import pyarrow.compute as pc
        cols.append(pc.binary_join_element_wise(pa.array(rng.integers(0, 1 << 40, n)).cast(pa.string()),
                                                pa.array(rng.integers(0, 1 << 30, n)).cast(pa.string()), " carefully final "))
        fields = [pa.field(nm, c.type, nullable=i >= schema.n_key + 2) for i, (nm, c) in enumerate(zip(names, cols))]
        return pa.Table.from_arrays(cols, schema=pa.schema(fields)), part, ship

    files = []
    exp_part = exp_ship = exp_seq = None
    for r in range(5):
        idx = np.arange(n_base, dtype=np.int64) if r == 0 else np.sort(rng.choice(n_base, n_upd, replace=False))
        seq0 = 0 if r == 0 else n_base + (r - 1) * n_upd
        tb, part, ship = run_table(idx, seq0)
        if r == 0:
            exp_part, exp_ship, exp_seq = part.copy(), ship.copy(), np.arange(n_base, dtype=np.int64)
        else:
            exp_part[idx] = part; exp_ship[idx] = ship; exp_seq[idx] = seq0 + np.arange(n_upd, dtype=np.int64)
        sink = pa.BufferOutputStream()
        pq.write_table(tb, sink, compression=codec, use_dictionary=True, data_page_version="1.0", data_page_size=160 << 10,
                       row_group_size=800_000, write_statistics=False, **({"compression_level": 1} if codec == "zstd" else {}))
        files.append((np.frombuffer(sink.getvalue(), np.uint8), r))
    return files, n_base + 4 * n_upd, {"l_partkey": exp_part, "l_shipdate": exp_ship, "_SEQUENCE_NUMBER": exp_seq}


# the keyword arguments c5_bucket passes to pyarrow.parquet.write_table, per codec (the test of this module holds them
# to the call in bench.py; the GPU tests read the page and row-group limits from here)
def c5_writer_args(codec):
    return dict(compression=codec, use_dictionary=True, data_page_version="1.0", data_page_size=160 << 10,
                row_group_size=800_000, write_statistics=False, **({"compression_level": 1} if codec == "zstd" else {}))
