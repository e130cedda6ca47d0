"""Cost of Parquet bloom filters (pg_parquet_encode_bloom) on a merged C3-shaped batch in HBM (pk + 20 BIGINT + 15
DOUBLE + 14 VARCHAR(24), half the cells NULL, 8 runs generated in HBM and merged with deduplicate; 3.60 M rows at the
default size).  Three cases, alternated off / four / all in every rep so that all see the same drift, uncompressed and
zstd-1:
  off   no bloom columns (pg_parquet_encode_compressed's bytes);
  four  four columns at the 1 MiB default (no ndv): i0 (BIGINT), _VALUE_KIND (TINYINT, written and hashed as INT32),
        d0 (DOUBLE), s0 (VARCHAR);
  all   'parquet.bloom.filter.enabled' = true: every file column, 1 MiB each.
Reported per case: pg_file_meta.ms_encode (the encoder's CUDA-event time) of every rep, the bytes the filters add
(file bytes minus the off case's), and in a torch.profiler run of its own the device time of k_pw_sbbf.  The card
name and power limit are read in the same run.
Usage: parquet_bloom_probe.py [c3_rows_per_run] [reps]"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import torch

import bench
from decode_kernels import gpu_identity
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.compact_rewriter import file_column_names, parquet_bloom_for_level
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader

rows_per_run = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
n_runs = 8
KERNEL = "k_pw_sbbf"

lib = N.init(0)
dev = torch.device("cuda:0")


def bloom_options(cols):
    arr = (N.PgParquetBloomColumn * max(len(cols), 1))(*[N.PgParquetBloomColumn(c, ndv, fpp) for c, ndv, fpp in cols])
    opts = N.PgParquetBloomOptions(len(cols), arr)
    opts._keep = arr
    return opts


def encode(handle, names, codec, bloom):
    opts = N.PgParquetWriteOptions(0, 0, 0)
    fh = C.c_uint64(0)
    N.check(lib.pg_parquet_encode_bloom(handle, names, 0, -1, C.byref(opts), codec, 1, C.byref(bloom), C.byref(fh)))
    meta = N.PgFileMeta()
    N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
    lib.pg_parquet_file_free(fh.value)
    return meta


def kernel_ms(handle, names, codec, bloom):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        encode(handle, names, codec, bloom)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if KERNEL in ev.key:
            return round((getattr(ev, "device_time_total", None) or ev.cuda_time_total) / 1e3, 3)
    return None


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
handle = mr._merge_h
names = file_column_names(c3)
arr = (C.c_char_p * len(names))(*[nm.encode() for nm in names])
col = {nm: i for i, nm in enumerate(names)}
cases = {"off": bloom_options([]),
         "four": bloom_options([(col[nm], 0, 0.01) for nm in ("i0", "_VALUE_KIND", "d0", "s0")]),
         "all": bloom_options(parquet_bloom_for_level(c3, {"parquet.bloom.filter.enabled": "true"}))}
res = {"rows": int(mr.device_batch().n_rows), "columns": len(names), "bloom_columns": {k: v.n_columns for k, v in cases.items()}}
for cname, codec in (("uncompressed", 0), ("zstd1", 6)):
    for b in cases.values():
        encode(handle, arr, codec, b)                                 # warm-up of every shape
    ms = {k: [] for k in cases}
    size = {}
    for _ in range(reps):
        for k, b in cases.items():
            m = encode(handle, arr, codec, b)
            ms[k].append(round(m.ms_encode, 3))
            size[k] = int(m.file_bytes)
    res[cname] = {k: {"ms_encode": ms[k], "ms_encode_min": min(ms[k]), "filter_bytes": size[k] - size["off"],
                      "kernel_ms": kernel_ms(handle, arr, codec, b)} for k, b in cases.items()}
    res[cname]["file_bytes_off"] = size["off"]
mr.close()
out["c3_merged"] = res
print(json.dumps(out, indent=1))
