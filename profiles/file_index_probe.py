"""Bloom-filter file index build (pg_bloom_filter_build) beside the Parquet encode of the same rows, on a merged
C3-shaped batch: the C3 row (pk + 20 BIGINT + 15 DOUBLE + 14 VARCHAR(24), half the cells NULL) with one INT field
added, 8 runs generated in HBM and merged with deduplicate.  Filters on one BIGINT, one INT, one DOUBLE and one STRING
column, at two sizings: the defaults (items 1 000 000, fpp 0.1: 599 071-byte filters that stay in L2) and items = the
rows of the file.  The build time is CUDA-event time on the default stream around the whole call (bit-set clear, job
table copy, k_bloom_build, copies of the filters back to the host); ms_encode is the encoder's own event time.  The
card name and power limit are read in the same run.  Usage: file_index_probe.py [rows_per_run] [reps]"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import numpy as np
import torch

import bench
from decode_kernels import gpu_identity
from paimon_b200 import _native as N
from paimon_b200.compact_rewriter import file_column_names
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader
from paimon_b200.types import DataField, KeyValueSchema, RowType
from paimon_b200 import datagen

rows_per_run = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
n_runs = 8

lib = N.init(0)
dev = torch.device("cuda:0")
c3 = datagen.schema_c3()
schema = KeyValueSchema.of(RowType(tuple(list(c3.value_type.fields) + [DataField("n0", "INT", True)])), ["pk"])
readers, keep = [], []
key_space = rows_per_run * n_runs // 2
for r in range(n_runs):
    cols, kp, _, _, _ = bench.gen_device_run(schema, r, rows_per_run, key_space, 0.5, 7, dev)
    readers.append(SortedRunReader.from_device(schema, rows_per_run, cols, keepalive=kp))
    keep.append(kp)
torch.cuda.synchronize()
mr = SortMergeReader.create_sort_merge_reader(readers, None, None, DeduplicateMergeFunction.factory().create())
mr.execute()
n_out = mr.device_batch().n_rows
names = file_column_names(schema)
arr = (C.c_char_p * len(names))(*[nm.encode() for nm in names])
indexed = {"i0": "BIGINT", "n0": "INT", "d0": "DOUBLE", "s0": "VARCHAR(24)"}
columns = [names.index(c) for c in indexed]


def encode(codec):
    fh = C.c_uint64(0)
    if codec is None:
        N.check(lib.pg_parquet_encode(mr._merge_h, arr, 0, -1, None, C.byref(fh)))
    else:
        N.check(lib.pg_parquet_encode_compressed(mr._merge_h, arr, 0, -1, None, codec, 1, C.byref(fh)))
    meta = N.PgFileMeta()
    N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
    lib.pg_parquet_file_free(fh.value)
    return meta.ms_encode


def bloom(items):
    specs = (N.PgBloomFilterSpec * len(columns))(*[N.PgBloomFilterSpec(c, items, 0.1) for c in columns])
    size = C.c_int64(0)
    N.check(lib.pg_bloom_filter_size(items, 0.1, C.byref(size), None))
    bufs = [np.empty(size.value, np.uint8) for _ in columns]
    outs = (C.c_void_p * len(columns))(*[b.ctypes.data for b in bufs])
    caps = (C.c_int64 * len(columns))(*[size.value] * len(columns))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(torch.cuda.default_stream())
    N.check(lib.pg_bloom_filter_build(mr._merge_h, 0, -1, len(columns), specs, outs, caps))
    e1.record(torch.cuda.default_stream())
    e1.synchronize()
    return e0.elapsed_time(e1), size.value


out = {"gpu": gpu_identity(0), "rows_out": int(n_out), "indexed_columns": indexed, "reps": reps}
for name, codec in (("parquet_uncompressed", None), ("parquet_zstd1", 6)):
    encode(codec)
    out[name + "_ms_encode"] = round(min(encode(codec) for _ in range(reps)), 3)
for name, items in (("bloom_default_items", 1_000_000), ("bloom_items_eq_rows", int(n_out))):
    bloom(items)
    ms, size = zip(*[bloom(items) for _ in range(reps)])
    out[name] = {"items": items, "filter_bytes": size[0], "ms": round(min(ms), 3), "ms_all": [round(x, 3) for x in ms]}
for name, items in (("bloom_default_items", 1_000_000), ("bloom_items_eq_rows", int(n_out))):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:   # a run of its own
        bloom(items)
        torch.cuda.synchronize()
    out[name]["kernels_ms"] = {ev.key[:60]: round((getattr(ev, "device_time_total", None) or ev.cuda_time_total) / 1e3, 3)
                               for ev in prof.key_averages()
                               if (getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0))}
mr.close()
print(json.dumps(out, indent=1))
