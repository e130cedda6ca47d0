"""ORC section decode from host bytes and from HBM-resident bytes: the C3 schema, 16 runs of one file each, written by
pg_orc_encode as NONE and as ZSTD.  For each codec it records the median PgSectionInfo.ms_decode (device events) over
`sections` decodes from host bytes, the same from device bytes, the wall time per section of an upload-pipelined loop
(FileUpload of section i + 1 in flight while section i decodes), and a hash of every decoded run (validity, values,
offsets, payload).  With --old LIB the host-byte decode of another build of libpaimon_gpu.so runs in the same call,
alternating with this tree's build (old, new, old, new, each in a process of its own); a build that refuses device
bytes reports so.  The ORC kernels' times come from a torch.profiler pass after the last run's timed sections.  One JSON line, with the card's
name and power limit read in the same call; with an output directory, also orc_device_probe.json there.
Usage: python profiles/orc_device_probe.py [--sections N] [--rows N] [--old LIB] [--out DIR]"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def run_hash(batch):
    from paimon_b200.columnar import is_varlen, unpack_validity
    import numpy as np
    h = hashlib.sha256()
    n = batch.n_rows
    for c in batch.columns:
        if c is None:
            continue
        h.update(unpack_validity(c.valid, n).tobytes())
        if is_varlen(c.type):
            o = np.asarray(c.offsets[:n + 1])
            h.update(o.tobytes())
            h.update(np.asarray(c.data[:o[-1]]).tobytes())
        else:
            h.update(np.asarray(c.data[:n]).tobytes())
    return h.hexdigest()[:16]


def worker(args):
    """One build (PAIMON_GPU_LIB) in a process of its own: encode, then decode."""
    import numpy as np
    import torch
    from paimon_b200 import _native as N
    from paimon_b200 import datagen
    from paimon_b200.compact_rewriter import KeyValueDataFileWriter
    from paimon_b200.format import FileUpload, read_section
    from paimon_b200.sort_merge_reader import SortedRunReader, _SchemaHandle

    def progress(msg):
        print(f"[{time.strftime('%H:%M:%S')}] {os.environ.get('PAIMON_GPU_LIB', 'this tree')}: {msg}", file=sys.stderr,
              flush=True)

    N.init(0)
    schema = datagen.schema_c3()
    runs = datagen.make_runs(schema, 16, args.rows, seed=3, null_prob=0.1)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for codec in ("none", "zstd"):
            files = []
            sh = _SchemaHandle(schema, 0)
            for i, run in enumerate(runs):
                path = os.path.join(tmp, f"r{i}.{codec}.orc")
                rd = SortedRunReader(schema, run)
                try:
                    KeyValueDataFileWriter(schema, path, level=1, file_format="orc", compression=codec).write(
                        rd._open(sh.handle))
                finally:
                    rd.close()
                files.append((np.fromfile(path, np.uint8), i))
            sh.close()
            progress(f"{codec}: 16 files written")
            file_hash = hashlib.sha256(b"".join(f.tobytes() for f, _ in files)).hexdigest()[:16]

            def section(fs, hashes=False):
                readers, info = read_section(schema, fs, 16, file_format="orc")
                hs = []
                for r in readers:
                    try:
                        if hashes:
                            hs.append(run_hash(r.read_batch()))
                    finally:
                        r.close()
                return info, hs

            res = {"file_bytes": int(sum(len(f) for f, _ in files)), "file_hash": file_hash}
            info, hs = section(files, True)
            res["runs_hash_host"] = hashlib.sha256("".join(hs).encode()).hexdigest()[:16]
            res["rows"] = int(info.n_rows)
            section(files)
            res["ms_decode_host"] = round(statistics.median(section(files)[0].ms_decode for _ in range(args.sections)), 3)
            progress(f"{codec}: host bytes {res['ms_decode_host']} ms")
            bufs = [torch.from_numpy(f).cuda() for f, _ in files]
            torch.cuda.synchronize()
            dev = [((b.data_ptr(), b.numel()), r) for b, (_, r) in zip(bufs, files)]
            try:
                info, hs = section(dev, True)
            except N.PaimonGpuError as e:
                res["device"] = f"refused: {e}"
                out[codec] = res
                continue
            res["runs_hash_device"] = hashlib.sha256("".join(hs).encode()).hexdigest()[:16]
            res["ms_decode_device"] = round(statistics.median(section(dev)[0].ms_decode for _ in range(args.sections)), 3)
            pinned = [(torch.from_numpy(f).pin_memory().numpy(), r) for f, r in files]
            up = FileUpload(pinned)
            t0 = time.perf_counter()
            for s in range(args.sections):
                nxt = FileUpload(pinned) if s + 1 < args.sections else None
                section(up.wait())
                up.close()
                up = nxt
            res["ms_section_pipelined"] = round((time.perf_counter() - t0) * 1e3 / args.sections, 3)
            progress(f"{codec}: device bytes {res['ms_decode_device']} ms, pipelined {res['ms_section_pipelined']} ms")
            if args.profile:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.sections):
                        section(dev)
                    torch.cuda.synchronize()
                res["kernel_ms"] = {ev.key.split("(")[0]: round(ev.device_time_total / 1e3 / args.sections, 3)
                                    for ev in prof.key_averages() if "k_orc" in ev.key}
            out[codec] = res
    print("RESULT " + json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sections", type=int, default=7)
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--old", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if args.worker:
        return worker(args)

    def spawn(lib, extra):
        env = dict(os.environ)
        if lib:
            env["PAIMON_GPU_LIB"] = lib
        cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--sections", str(args.sections), "--rows",
               str(args.rows)] + extra
        p = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, text=True)      # (progress goes to stderr as it comes)
        line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
        if p.returncode or not line:
            raise SystemExit(f"worker failed ({lib or 'this tree'}):\n{p.stdout[-3000:]}")
        return json.loads(line[0][7:])

    out = {"card": card(), "runs": 16, "rows": args.rows, "sections": args.sections, "builds": []}
    order = [("old", args.old), ("new", None)] * 2 if args.old else [("new", None)]
    for i, (name, lib) in enumerate(order):
        # (the last run of this tree's build adds the torch.profiler pass, after its timed sections)
        out["builds"].append({"build": name, **spawn(lib, ["--profile"] if i == len(order) - 1 else [])})
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "orc_device_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
