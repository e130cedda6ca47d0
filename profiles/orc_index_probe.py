"""Cost of the ORC row index (pg_orc_encode_indexed) on a merged C3-shaped batch in HBM (pk + 20 BIGINT + 15 DOUBLE +
14 VARCHAR(24), half the cells NULL, 8 runs generated in HBM and merged with deduplicate).  Three shapes, alternated
plain / stride 10000 / stride 10000 + 3 bloom filters (a BIGINT, a DOUBLE and a VARCHAR column, fpp 0.01) so that all
see the same drift, for both codecs (NONE, ZSTD-1).  Reported per case: pg_file_meta.ms_encode (the encoder's
CUDA-event time) of every rep, the index bytes (file bytes minus the plain file's), and in a torch.profiler run of its
own the device time of k_oe_count, k_pw_stats and k_oe_bloom.  The card name and power limit are read in the same run.
Usage: orc_index_probe.py [rows_per_run] [reps]"""
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
from paimon_b200.compact_rewriter import file_column_names
from paimon_b200.merge_function import DeduplicateMergeFunction
from paimon_b200.sort_merge_reader import SortedRunReader, SortMergeReader
from paimon_b200.types import orc_column_type

rows_per_run = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
n_runs = 8
KERNELS = ("k_oe_count", "k_pw_stats", "k_oe_bloom")

lib = N.init(0)
dev = torch.device("cuda:0")


def encode(handle, names, opts, index):
    fh = C.c_uint64(0)
    if index is None:
        N.check(lib.pg_orc_encode(handle, names, 0, -1, C.byref(opts), C.byref(fh)))
    else:
        N.check(lib.pg_orc_encode_indexed(handle, names, 0, -1, C.byref(opts), C.byref(index), C.byref(fh)))
    meta = N.PgFileMeta()
    N.check(lib.pg_parquet_file_meta(fh.value, C.byref(meta)))
    lib.pg_parquet_file_free(fh.value)
    return meta


def kernel_ms(*args):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        encode(*args)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                out[k] = round((getattr(ev, "device_time_total", None) or ev.cuda_time_total) / 1e3, 3)
    return out


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

fields = c3.file_fields()
names = file_column_names(c3)
arr = (C.c_char_p * len(names))(*[nm.encode() for nm in names])
types = (N.PgOrcColumnType * len(fields))(*[N.PgOrcColumnType(*orc_column_type(f.type)) for f in fields])
first = {}
for i, f in enumerate(fields[c3.n_key + 2:]):
    first.setdefault(f.type.split("(")[0], c3.n_key + 2 + i)
bloom = (C.c_int32 * 3)(first["BIGINT"], first["DOUBLE"], first["VARCHAR"])
shapes = {"plain": None, "stride10000": N.PgOrcIndexOptions(10000, 0, None, 0.01),
          "stride10000_bloom3": N.PgOrcIndexOptions(10000, 3, bloom, 0.01)}

out = {"gpu": gpu_identity(0), "reps": reps, "rows": int(mr.device_batch().n_rows), "columns": len(names),
       "bloom_columns": [names[c] for c in bloom]}
for cname, codec in (("none", 0), ("zstd1", 5)):
    opts = N.PgOrcWriteOptions(0, codec, 1, 0, types)
    for ix in shapes.values():
        encode(handle, arr, opts, ix)                                  # warm-up of every shape
    ms = {k: [] for k in shapes}
    size = {}
    for _ in range(reps):
        for k, ix in shapes.items():
            m = encode(handle, arr, opts, ix)
            ms[k].append(round(m.ms_encode, 3))
            size[k] = int(m.file_bytes)
    out[cname] = {k: {"ms_encode": ms[k], "ms_encode_min": min(ms[k]), "index_bytes": size[k] - size["plain"],
                      "kernels_ms": kernel_ms(handle, arr, opts, ix)} for k, ix in shapes.items()}
    out[cname]["file_bytes_plain"] = size["plain"]
mr.close()
print(json.dumps(out, indent=1))
