"""Where the GPU idles during the bench's C3 step: read_section -> rebind -> execute, on one GPU.

Builds the bench's C3 section the way profiles/decode_kernels.py does (bench.device_parquet_files), warms up, then runs
--steps full steps (the calls of bench.py's one_step) under torch.profiler with CUDA activities.  A one-element torch
kernel on the decode stream marks the start of each step on the device.  Per step it reports, from the trace:

    ms_decode           the decode's own CUDA-event time (pg_section_info.ms_decode)
    decode_first/last   first and last decode kernel (k_pq_*)
    idle_before_ms      step start -> first decode kernel: footers, their parse, the chunk tables, the table uploads
    decode_gaps_ms      device idle between the first and the last decode kernel, every stream together (the
                        read-backs and the host work behind them), and each gap above 10 us with its neighbours
    decode_to_merge_ms  last decode activity -> first merge activity (the end of the decode, rebind)
    merge_gaps_ms       device idle inside the merge, each gap above 10 us with its neighbours (the size read-back)
    ms_total_merge      the merge's own CUDA-event time (pg_stats.ms_total)

and the GPU's name and power limit.  Each build runs in a subprocess of its own (PAIMON_GPU_LIB selects it), so that
several builds can be compared in one call, alternating:

    python profiles/step_timeline.py [--lib NAME=PATH ...] [--rounds 2] [--steps 5] [--rows N] [--out DIR]
                                     [--host-timing NAME=PATH]

--lib defaults to the in-tree build.  --host-timing runs a build made with EXTRA_DEFS=-DPG_HOST_TIMING (no profiler)
and averages the host phase times it prints per call.  Writes under DIR (default: step_timeline/ in the system's
temporary directory) summary.json and, per build and round, the worker's JSON and trace; prints one table.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
os.environ.setdefault("PG_RUN_CACHE_BYTES", str(64 << 30))

GAP_US = 10.0


def busy_gaps(acts, t0, t1):
    """Idle intervals of the device inside [t0, t1] (us): where no activity of any stream runs."""
    gaps, cur, prev = [], t0, None
    for a in sorted(acts, key=lambda a: a["ts"]):
        if a["ts"] + a["dur"] <= t0 or a["ts"] >= t1:
            continue
        if a["ts"] > cur:
            gaps.append((cur, a["ts"], prev, a["name"]))
        if a["ts"] + a["dur"] > cur:
            cur, prev = a["ts"] + a["dur"], a["name"]
    return gaps


def short(name):
    n = name.split("(")[0].replace("void ", "").replace("pg::", "").replace("(anonymous namespace)::", "")
    return n[:40]


def analyse(trace_path, marker):
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    acts = sorted(({"name": e["name"], "ts": float(e["ts"]), "dur": float(e.get("dur", 0)),
                    "stream": e.get("args", {}).get("stream")}
                   for e in ev if e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")), key=lambda a: a["ts"])
    # the step marker: torch's fill kernel on a one-element tensor, the only torch kernel of a step
    marks = [a for a in acts if marker in a["name"]]
    steps = []
    for i, m in enumerate(marks):
        end = marks[i + 1]["ts"] if i + 1 < len(marks) else float("inf")
        win = [a for a in acts if m["ts"] + m["dur"] <= a["ts"] < end and a is not m]
        dec = [a for a in win if "k_pq" in a["name"]]
        if not dec:
            continue
        d0 = dec[0]["ts"]
        d1 = max(a["ts"] + a["dur"] for a in dec)
        # the decode ends with its error-word read-back; the merge starts with the first activity after it
        after = [a for a in win if a["ts"] >= d1]
        dec_end = after[0]["ts"] + after[0]["dur"] if after else d1
        merge = after[1:]
        m0 = merge[0]["ts"] if merge else dec_end
        m1 = max((a["ts"] + a["dur"] for a in merge), default=m0)
        dg = busy_gaps(win, d0, d1)
        mg = busy_gaps(win, m0, m1)
        steps.append({
            "decode_first": short(dec[0]["name"]), "decode_last": short(max(dec, key=lambda a: a["ts"] + a["dur"])["name"]),
            "idle_before_ms": (d0 - (m["ts"] + m["dur"])) / 1e3,
            "decode_span_ms": (d1 - d0) / 1e3,
            "decode_gaps_ms": sum(b - a for a, b, _, _ in dg) / 1e3,
            "decode_gap_list": [[round((b - a) / 1e3, 3), short(p or ""), short(n)] for a, b, p, n in dg if b - a > GAP_US],
            "decode_to_merge_ms": (m0 - d1) / 1e3,
            "merge_span_ms": (m1 - m0) / 1e3,
            "merge_gaps_ms": sum(b - a for a, b, _, _ in mg) / 1e3,
            "merge_gap_list": [[round((b - a) / 1e3, 3), short(p or ""), short(n)] for a, b, p, n in mg if b - a > GAP_US],
        })
    return steps


def worker(args):
    import ctypes as C

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from decode_kernels import gpu_identity
    from paimon_b200 import _native as N
    from paimon_b200.format import read_section
    from paimon_b200.sort_merge_reader import SortMergeReader

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    w = bench.WORKLOADS["c3"]
    rows = args.rows or w["rows"]
    schema = bench.make_schema("c3")
    spec = bench.make_spec("c3", schema)
    lib = N.init(0)
    _, images, _, _ = bench.device_parquet_files("c3", schema, rows, dev, 100, lib)
    files = [(img, r) for r, img in enumerate(images)]
    rd = SortMergeReader([], spec, None, 0, schema=schema)
    dstream = C.c_void_p(0)
    N.check(lib.pg_thread_stream(C.byref(dstream)))
    ext_dec = torch.cuda.ExternalStream(dstream.value or 0, device=dev)
    flag = torch.zeros(1, device=dev)

    def one_step():
        with torch.cuda.stream(ext_dec):
            flag.fill_(1.0)                                  # the step's start on the device
        readers, info = read_section(schema, files, w["n_runs"], 0)
        rd.rebind(readers)
        rd.execute()
        st = rd.stats()
        for r in readers:
            r.close()
        rd.readers = []
        return info, st

    for _ in range(args.warmup):
        one_step()
    torch.cuda.synchronize()
    out = {"gpu": gpu_identity(0), "rows": rows, "lib": os.environ.get("PAIMON_GPU_LIB", "in-tree")}
    if args.no_profile:
        res = [one_step() for _ in range(args.steps)]
        torch.cuda.synchronize()
        out["ms_decode"] = [i.ms_decode for i, _ in res]
    else:
        res = []
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                res.append(one_step())
            torch.cuda.synchronize()
        trace = args.worker_out + ".pt.trace.json"
        prof.export_chrome_trace(trace)
        steps = analyse(trace, "FillFunctor")
        for s, (info, st) in zip(steps, res):
            s["ms_decode"] = info.ms_decode
            s["ms_total_merge"] = st.ms_total
        out["steps"] = steps
    rd.close()
    with open(args.worker_out + ".json", "w") as f:
        json.dump(out, f, indent=1)


HOST_LINE = re.compile(r"\[host timing\] ([^:]+):(.*) total ([0-9.]+)")


def run_worker(args, name, path, tag, no_profile=False):
    env = dict(os.environ)
    if path:
        env["PAIMON_GPU_LIB"] = os.path.abspath(path)
    base = os.path.join(args.out, tag)
    cmd = [sys.executable, os.path.abspath(__file__), "--worker-out", base, "--steps", str(args.steps),
           "--warmup", str(args.warmup)] + (["--rows", str(args.rows)] if args.rows else []) + \
          (["--no-profile"] if no_profile else [])
    p = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-4000:] + p.stderr[-4000:])
        raise SystemExit(f"{name}: worker failed ({p.returncode})")
    with open(base + ".json") as f:
        res = json.load(f)
    res["name"] = name
    if no_profile:
        phases = {}
        for line in p.stderr.splitlines():
            mt = HOST_LINE.search(line)
            if not mt:
                continue
            toks = mt.group(2).split()
            calls = phases.setdefault(mt.group(1), [])
            calls.append({toks[i]: float(toks[i + 1]) for i in range(0, len(toks) - 1, 2)} | {"total": float(mt.group(3))})
        # the timed steps are the last ones printed
        res["host_phases_ms"] = {who: {k: sum(c.get(k, 0.0) for c in cs[-args.steps:]) / len(cs[-args.steps:])
                                       for k in cs[-1]} for who, cs in phases.items()}
    return res


def mean(xs):
    return sum(xs) / len(xs) if xs else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH",
                    help="a build to measure (repeatable; default: the in-tree build)")
    ap.add_argument("--host-timing", action="append", default=[], metavar="NAME=PATH",
                    help="a -DPG_HOST_TIMING build: host phase times per call (no profiler)")
    ap.add_argument("--rounds", type=int, default=2, help="rounds of the builds, alternating A B A B")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=None, help="total input rows (default: the bench's C3 size)")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "step_timeline"))
    ap.add_argument("--worker-out", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--no-profile", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker_out:
        return worker(args)

    os.makedirs(args.out, exist_ok=True)
    libs = [tuple(x.split("=", 1)) for x in args.lib] or [("in-tree", None)]
    results = []
    for rnd in range(args.rounds):
        for name, path in libs:
            r = run_worker(args, name, path, f"{name}_r{rnd}")
            r["round"] = rnd
            results.append(r)
    host = [run_worker(args, name, path, f"{name}_host", no_profile=True) for name, path in
            (tuple(x.split("=", 1)) for x in args.host_timing)]

    keys = ["ms_decode", "idle_before_ms", "decode_gaps_ms", "decode_span_ms", "decode_to_merge_ms", "merge_gaps_ms",
            "merge_span_ms", "ms_total_merge"]
    table = []
    for r in results:
        row = {"build": r["name"], "round": r["round"]}
        for k in keys:
            row[k] = mean([s[k] for s in r["steps"]])
        row["host_idle_in_decode_ms"] = row["idle_before_ms"] + row["decode_gaps_ms"]
        table.append(row)
    summary = {"gpu": results[0]["gpu"], "rows": results[0]["rows"], "steps_per_run": args.steps, "table": table,
               "runs": results, "host_timing": host}
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)

    print(json.dumps(summary["gpu"]), f"rows={summary['rows']} steps per run={args.steps}")
    cols = ["ms_decode", "idle_before_ms", "decode_gaps_ms", "host_idle_in_decode_ms", "decode_to_merge_ms",
            "merge_gaps_ms", "ms_total_merge"]
    print(f"{'build':<12}{'rnd':>4}" + "".join(f"{c:>24}" for c in cols))
    for row in table:
        print(f"{row['build']:<12}{row['round']:>4}" + "".join(f"{row[c]:>24.3f}" for c in cols))
    for r in results:
        s = r["steps"][-1]
        print(f"{r['name']} r{r['round']} last step: first {s['decode_first']}, last {s['decode_last']}; "
              f"decode gaps {s['decode_gap_list']}; merge gaps {s['merge_gap_list']}")
    for h in host:
        for who, ph in h["host_phases_ms"].items():
            print(f"{h['name']} host phases, {who}: " + ", ".join(f"{k} {v:.3f}" for k, v in ph.items()))


if __name__ == "__main__":
    main()
