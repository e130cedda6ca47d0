"""Cost of the Parquet page index (pg_parquet_write_options.page_index = 1) on two batches in HBM: a merged C3-shaped
batch (pk + 20 BIGINT + 15 DOUBLE + 14 VARCHAR(24), half the cells NULL, 8 runs generated in HBM and merged with
deduplicate) and a C5 (lineitem-shaped) batch of one run (DECIMAL / DATE in their INT64 / INT32 form, four STRING
columns).  Both codecs (uncompressed, zstd-1), the index off and on alternated off / on / off / on so that both see the
same drift.  Reported per case: pg_file_meta.ms_encode (the encoder's CUDA-event time) of every rep, the index bytes
(file bytes on minus off), and in a torch.profiler run of its own the device time of k_pw_stats and
k_pw_minmax_bytes.  The card name and power limit are read in the same run.
Usage: page_index_probe.py [c3_rows_per_run] [c5_rows] [reps]"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import torch

import bench
from decode_kernels import gpu_identity
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import Column, KeyValueBatch
from paimon_b200.compact_rewriter import file_column_names
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader, _SchemaHandle
from paimon_b200.types import DataField, KeyValueSchema, RowType

rows_per_run = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
c5_rows = int(sys.argv[2]) if len(sys.argv) > 2 else 4_000_000
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
n_runs = 8
KERNELS = ("k_pw_stats", "k_pw_minmax_bytes")

lib = N.init(0)
dev = torch.device("cuda:0")


def c5_batch(n, seed=5):
    fields = [DataField("l_orderkey", "BIGINT", False), DataField("l_linenumber", "INT", False),
              DataField("l_partkey", "BIGINT", True), DataField("l_suppkey", "BIGINT", True),
              DataField("l_quantity", "BIGINT", True), DataField("l_extendedprice", "BIGINT", True),
              DataField("l_discount", "BIGINT", True), DataField("l_tax", "BIGINT", True),
              DataField("l_returnflag", "STRING", True), DataField("l_linestatus", "STRING", True),
              DataField("l_shipdate", "INT", True), DataField("l_commitdate", "INT", True),
              DataField("l_receiptdate", "INT", True), DataField("l_shipinstruct", "STRING", True),
              DataField("l_shipmode", "STRING", True), DataField("l_comment", "STRING", True)]
    schema = KeyValueSchema.of(RowType(tuple(fields)), ["l_orderkey", "l_linenumber"])
    rng = np.random.default_rng(seed)
    idx = np.arange(n, dtype=np.int64)
    ok, ln = idx // 4, (idx % 4 + 1).astype(np.int32)
    flags = [np.array([b"A", b"N", b"R"]), np.array([b"F", b"O"])]
    instr = np.array([b"DELIVER IN PERSON", b"COLLECT COD", b"NONE", b"TAKE BACK RETURN"])
    modes = np.array([b"REG AIR", b"AIR", b"RAIL", b"SHIP", b"TRUCK", b"MAIL", b"FOB"])
    ship = rng.integers(8000, 10600, n).astype(np.int32)
    cols = [pa.array(ok), pa.array(ln), pa.array(idx), pa.array(np.zeros(n, np.int8)), pa.array(ok), pa.array(ln),
            pa.array(rng.integers(1, 20_000_000, n)), pa.array(rng.integers(1, 1_000_000, n))]
    cols += [pa.array(rng.integers(100, 5_000_000, n)) for _ in range(4)]
    cols += [pa.array(flags[0][rng.integers(0, 3, n)]).cast(pa.string()),
             pa.array(flags[1][rng.integers(0, 2, n)]).cast(pa.string())]
    cols += [pa.array(ship), pa.array(ship + 30), pa.array(ship + 45)]
    cols += [pa.array(instr[rng.integers(0, 4, n)]).cast(pa.string()),
             pa.array(modes[rng.integers(0, 7, n)]).cast(pa.string())]
    cols.append(pc.binary_join_element_wise(pa.array(rng.integers(0, 1 << 40, n)).cast(pa.string()),
                                            pa.array(rng.integers(0, 1 << 30, n)).cast(pa.string()), " carefully final "))
    out = []
    for t, a in zip(schema.physical_types(), cols):
        a = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
        if a.type == pa.string():
            bufs = a.buffers()
            off = np.frombuffer(bufs[1], np.int32, len(a) + 1, a.offset * 4).copy()
            out.append(Column(t, np.frombuffer(bufs[2], np.uint8, off[-1]).copy(), off, None))
        else:
            out.append(Column(t, a.to_numpy(zero_copy_only=False), None, None))
    return schema, KeyValueBatch(schema, out)


def encode(handle, names, codec, page_index):
    opts = N.PgParquetWriteOptions(0, 0, page_index)
    fh = C.c_uint64(0)
    if codec is None:
        N.check(lib.pg_parquet_encode(handle, names, 0, -1, C.byref(opts), C.byref(fh)))
    else:
        N.check(lib.pg_parquet_encode_compressed(handle, names, 0, -1, C.byref(opts), codec, 1, C.byref(fh)))
    meta = N.PgFileMeta()
    N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
    lib.pg_parquet_file_free(fh.value)
    return meta


def kernel_ms(handle, names, codec, page_index):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        encode(handle, names, codec, page_index)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                out[k] = round((getattr(ev, "device_time_total", None) or ev.cuda_time_total) / 1e3, 3)
    return out


def measure(label, schema, handle, n_rows):
    names = file_column_names(schema)
    arr = (C.c_char_p * len(names))(*[nm.encode() for nm in names])
    res = {"rows": int(n_rows), "columns": len(names)}
    for cname, codec in (("uncompressed", None), ("zstd1", 6)):
        encode(handle, arr, codec, 0)
        encode(handle, arr, codec, 1)                                 # warm-up of both shapes
        ms = {0: [], 1: []}
        size = {}
        for _ in range(reps):
            for pi in (0, 1):
                m = encode(handle, arr, codec, pi)
                ms[pi].append(round(m.ms_encode, 3))
                size[pi] = int(m.file_bytes)
        res[cname] = {"ms_encode_off": ms[0], "ms_encode_on": ms[1],
                      "ms_encode_off_min": min(ms[0]), "ms_encode_on_min": min(ms[1]),
                      "file_bytes_off": size[0], "index_bytes": size[1] - size[0],
                      "kernels_ms_off": kernel_ms(handle, arr, codec, 0),
                      "kernels_ms_on": kernel_ms(handle, arr, codec, 1)}
    out[label] = res


out = {"gpu": gpu_identity(0), "reps": reps}

c3 = datagen.schema_c3()
readers = []
key_space = rows_per_run * n_runs // 2
for r in range(n_runs):
    cols, kp, _, _, _ = bench.gen_device_run(c3, r, rows_per_run, key_space, 0.5, 7, dev)
    readers.append(SortedRunReader.from_device(c3, rows_per_run, cols, keepalive=kp))
torch.cuda.synchronize()
mr = SortMergeReader.create_sort_merge_reader(readers, None, None, DeduplicateMergeFunction.factory().create())
mr.execute()
measure("c3_merged", c3, mr._merge_h, mr.device_batch().n_rows)
mr.close()

c5, batch = c5_batch(c5_rows)
sh = _SchemaHandle(c5, 0)
rd = SortedRunReader(c5, batch)
try:
    measure("c5_run", c5, rd._open(sh.handle), batch.n_rows)
finally:
    rd.close()
    sh.close()
print(json.dumps(out, indent=1))
