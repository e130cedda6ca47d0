"""Parquet codec 5 (Hadoop-framed LZ4) against Snappy on the same page bodies: one C5 bucket (bench.c5_bucket: 15.6 M
lineitem-shaped rows in 5 runs, dictionary on, page V1, 160 KiB pages) written uncompressed, then every page body
recompressed once as codec 5 and once as Snappy (tests/lz4_parquet.to_hadoop_lz4), both decoded from HBM-resident file
bytes.  Prints the section decode stage (PgSectionInfo.ms_decode, device events) and the per-kernel CUDA time of the
page decompression kernel (torch.profiler) for each, with the card name and power limit read in the same run, as one
JSON line; with an output directory, also as lz4_probe.json there.
Usage: python profiles/lz4_probe.py [steps] [output directory]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from lz4_parquet import LZ4, SNAPPY, to_hadoop_lz4  # noqa: E402
from paimon_b200.format import FileUpload, read_section  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def decode(schema, dev_files, steps):
    ms, kernel_ms = [], {}
    for it in range(2 + steps):
        readers, info = read_section(schema, dev_files, 5)
        for r in readers:
            r.close()
        if it >= 2:
            ms.append(info.ms_decode)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            readers, _ = read_section(schema, dev_files, 5)
            for r in readers:
                r.close()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if ev.key.startswith("k_pq") or "pg::k_pq" in ev.key:
            kernel_ms[ev.key.split("(")[0]] = round(ev.device_time_total / 1e3 / steps, 3)
    return ms, kernel_ms, info


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    torch.cuda.init()
    schema = bench.schema_c5()
    files, n_in, _ = bench.c5_bucket(schema, "none")
    out = {"card": card(), "rows": n_in}
    for name, codec in (("lz4", LZ4), ("snappy", SNAPPY)):
        blobs = [(np.frombuffer(to_hadoop_lz4(bytes(b), codec), np.uint8), r) for b, r in files]
        up = FileUpload(blobs)
        try:
            dev_files = up.wait()
            ms, kernels, info = decode(schema, dev_files, steps)
        finally:
            up.close()
        out[name] = {"file_bytes": int(sum(len(b) for b, _ in blobs)), "pages": info.n_data_pages,
                     "ms_decode_median": round(float(np.median(ms)), 3), "ms_decode_min": round(min(ms), 3),
                     "kernels_ms_per_section": kernels}
    out["card_after"] = card()
    print(json.dumps(out))
    if len(sys.argv) > 2:
        os.makedirs(sys.argv[2], exist_ok=True)
        with open(os.path.join(sys.argv[2], "lz4_probe.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
