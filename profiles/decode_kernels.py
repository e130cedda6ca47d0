"""Per-kernel profile of the C3 decode stage on one GPU.

Builds the bench's C3 section (the same device-encoded Parquet files, through bench.device_parquet_files and
bench.make_schema), warms up, then decodes it --reps times under torch.profiler with CUDA activities.  Only the decode
runs here, no merge, so every kernel in the capture belongs to the decode stage.

    python profiles/decode_kernels.py [--rows N] [--reps 3] [--out DIR]

Writes under DIR (default: decode_kernels/ in the system's temporary directory):
    kernels.csv    per kernel name and stream: launches per decode, total / mean ms per decode
    summary.json   the same plus, per decode: the stage span (first to last decode kernel), the side-stream span
                   (fork to join: first to last kernel on the side stream), the main-stream expansion span, the idle
                   gaps on the main decode stream between consecutive kernels, the GPU name and power limit
    trace.pt.trace.json  the raw capture (ignored by git)
and prints the tables.
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("PG_RUN_CACHE_BYTES", str(64 << 30))


def gpu_identity(index):
    """Name, power limit and max SM clock as nvidia-smi reports them (read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clock}
    except Exception as e:                                   # noqa: BLE001 (no nvidia-smi: report what torch knows)
        import torch
        return {"name": torch.cuda.get_device_name(index), "power_limit": None, "error": repr(e)[:200]}


def decode_windows(kernels):
    """Split the decode kernels into one list per decode: every decode starts with the page walk's count pass."""
    wins, cur = [], []
    for k in kernels:
        if "k_pq_walk<false>" in k["name"] and cur:
            wins.append(cur)
            cur = []
        cur.append(k)
    if cur:
        wins.append(cur)
    return wins


def short(name):
    n = name.split("(")[0]
    return n.replace("pg::", "").replace("void ", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=None, help="total input rows (default: the bench's C3 size)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "decode_kernels"))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from paimon_b200 import _native as N
    from paimon_b200.format import read_section

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    w = bench.WORKLOADS["c3"]
    rows = args.rows or w["rows"]
    schema = bench.make_schema("c3")
    lib = N.init(0)
    _, images, _, _ = bench.device_parquet_files("c3", schema, rows, dev, 100, lib)
    files = [(img, r) for r, img in enumerate(images)]

    def decode():
        readers, info = read_section(schema, files, w["n_runs"], 0)
        for r in readers:
            r.close()
        return info

    for _ in range(args.warmup):
        decode()
    torch.cuda.synchronize()
    infos = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            infos.append(decode())
        torch.cuda.synchronize()
    os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out, "trace.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = json.load(f)["traceEvents"]
    kernels = sorted(({"name": e["name"], "ts": float(e["ts"]), "dur": float(e["dur"]),
                       "stream": e.get("args", {}).get("stream")}
                      for e in ev if e.get("cat") == "kernel" and "k_pq" in e.get("name", "")),
                     key=lambda k: k["ts"])
    wins = decode_windows(kernels)
    n = len(wins)

    per = collections.defaultdict(lambda: {"launches": 0, "ms": 0.0})
    for k in kernels:
        key = (short(k["name"]), k["stream"])
        per[key]["launches"] += 1
        per[key]["ms"] += k["dur"] / 1e3
    main_stream = wins[0][0]["stream"] if wins else None
    table = [{"kernel": name, "stream": s, "side": s != main_stream, "launches_per_decode": v["launches"] / n,
              "ms_per_decode": v["ms"] / n} for (name, s), v in per.items()]
    table.sort(key=lambda r: -r["ms_per_decode"])

    spans = []
    for win in wins:
        t0 = win[0]["ts"]
        t1 = max(k["ts"] + k["dur"] for k in win)
        side = [k for k in win if k["stream"] != main_stream]
        mains = [k for k in win if k["stream"] == main_stream]
        exp_main = [k for k in mains if "k_pq_expand" in k["name"]]
        gaps = [(b["ts"] - (a["ts"] + a["dur"])) / 1e3 for a, b in zip(mains, mains[1:])]
        spans.append({
            "stage_ms": (t1 - t0) / 1e3,
            "side_fork_to_join_ms": ((max(k["ts"] + k["dur"] for k in side) - min(k["ts"] for k in side)) / 1e3
                                     if side else 0.0),
            "main_expand_ms": sum(k["dur"] for k in exp_main) / 1e3,
            "main_stream_gaps_ms": [round(g, 3) for g in gaps],
            "main_stream_idle_ms": sum(max(g, 0.0) for g in gaps),
        })
    summary = {
        "gpu": gpu_identity(0),
        "rows": rows,
        "decodes": n,
        "pages": int(infos[-1].n_data_pages),
        "launches": int(infos[-1].launches),
        "ms_decode_events": [round(i.ms_decode, 3) for i in infos],
        "kernels": table,
        "per_decode": spans,
    }
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    with open(os.path.join(args.out, "kernels.csv"), "w") as f:
        f.write("kernel,stream,side,launches_per_decode,ms_per_decode\n")
        for r in table:
            f.write(f"{r['kernel']},{r['stream']},{int(r['side'])},{r['launches_per_decode']:g},{r['ms_per_decode']:.3f}\n")

    print(json.dumps(summary["gpu"]), f"rows={rows} pages={summary['pages']} launches={summary['launches']}")
    print("ms_decode (CUDA events):", summary["ms_decode_events"])
    print(f"{'kernel':<28}{'stream':>8}{'side':>6}{'launches':>10}{'ms':>10}")
    for r in table:
        print(f"{r['kernel']:<28}{str(r['stream']):>8}{int(r['side']):>6}{r['launches_per_decode']:>10g}"
              f"{r['ms_per_decode']:>10.3f}")
    for i, s in enumerate(spans):
        print(f"decode {i}: stage {s['stage_ms']:.3f} ms, side fork->join {s['side_fork_to_join_ms']:.3f} ms, "
              f"main expand {s['main_expand_ms']:.3f} ms, main-stream idle {s['main_stream_idle_ms']:.3f} ms "
              f"(gaps {s['main_stream_gaps_ms']})")


if __name__ == "__main__":
    main()
