"""Compaction output encode, uncompressed vs zstd-1 on the device, on a merged C5 bucket (bench.c5_bucket): decode the
bucket's files, merge them, then encode the merged batch both ways.  Reports encode ms, uncompressed page GB/s, file
bytes and ratio, per-kernel device times from torch.profiler, and libzstd level 1 over the same page bodies on every
host core (the bar the device compressor is measured against).  The card name and power limit are read in the same
run.  Usage: encode_probe.py [reps]"""
import ctypes as C
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import pyarrow as pa
import torch

import bench
from decode_kernels import gpu_identity
from paimon_b200 import _native as N
from paimon_b200.compact_rewriter import file_column_names
from paimon_b200.format import read_section
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.sort_merge_reader import SortMergeReader
from test_gpu_parquet_write_zstd import pages_of

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
lib = N.init(0)
schema = bench.schema_c5()
files, n_in, _ = bench.c5_bucket(schema, "none")
readers, info = read_section(schema, files, 5)
mr = SortMergeReader.create_sort_merge_reader(readers, None, None, DeduplicateMergeFunction.factory().create())
mr.execute()
n_out = mr.device_batch().n_rows
names = file_column_names(schema)
arr = (C.c_char_p * len(names))(*[nm.encode() for nm in names])


def encode(codec):
    fh = C.c_uint64(0)
    if codec is None:
        N.check(lib.pg_parquet_encode(mr._merge_h, arr, 0, -1, None, C.byref(fh)))
    else:
        N.check(lib.pg_parquet_encode_compressed(mr._merge_h, arr, 0, -1, None, codec, 1, C.byref(fh)))
    meta = N.PgFileMeta()
    N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
    buf = np.zeros(meta.file_bytes, np.uint8)
    N.check(lib.pg_parquet_file_fetch(fh.value, buf.ctypes.data, meta.file_bytes))
    lib.pg_parquet_file_free(fh.value)
    return meta, bytes(buf)


out = {"gpu": gpu_identity(0), "rows_in": int(n_in), "rows_out": int(n_out), "host_cores": os.cpu_count()}
bodies = None
for name, codec in (("uncompressed", None), ("zstd-1", 6)):
    encode(codec)                                                        # warm-up
    ms = []
    for _ in range(reps):
        meta, file_bytes = encode(codec)
        ms.append(meta.ms_encode)
    pages = pages_of(file_bytes)
    if codec is None:
        bodies = [b for _, b in pages]
    raw = sum(u for u, _ in pages)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        encode(codec)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t:
            kernels[ev.key[:60]] = round(t / 1e3, 3)
    out[name] = {"encode_ms": round(min(ms), 3), "encode_ms_all": [round(x, 3) for x in ms],
                 "launches": int(meta.launches), "page_bytes": raw, "file_bytes": len(file_bytes),
                 "page_GB_per_s": round(raw / (min(ms) * 1e-3) / 1e9, 2), "kernels_ms": kernels}
out["ratio_uncompressed_over_zstd"] = round(out["uncompressed"]["file_bytes"] / out["zstd-1"]["file_bytes"], 3)

# libzstd level 1 over the same page bodies, every host core
codec = pa.Codec("zstd", compression_level=1)
best = None
for _ in range(reps):
    t0 = time.perf_counter()
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        sizes = list(ex.map(lambda b: len(codec.compress(b, asbytes=True)), bodies))
    dt = time.perf_counter() - t0
    best = dt if best is None else min(best, dt)
raw = sum(len(b) for b in bodies)
out["libzstd1_all_cores"] = {"ms": round(best * 1e3, 2), "GB_per_s": round(raw / best / 1e9, 2), "bytes": sum(sizes)}
out["device_zstd_over_libzstd1_bytes"] = round(sum(len(f) for _, f in pages_of(encode(6)[1])) / sum(sizes), 3)
mr.close()
print(json.dumps(out, indent=1))
