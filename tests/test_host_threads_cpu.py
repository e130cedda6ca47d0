"""The Parquet footer and ORC tail parsers (parquet_meta.cc, orc_meta.cc) on 8 threads at once, in a host build under
ThreadSanitizer (tests/native/threads_host_check.cc).  The section decoders parse on whatever thread calls them, so
reader threads of one process parse footers and tails at the same time; the ORC tail inflates zlib and zstd metadata
through per-thread tables.  Every concurrent parse must equal the sequential parse of the same file, on inputs shared by
every thread and on inputs of one thread each, and ThreadSanitizer must report nothing."""
import os
import struct
import subprocess

import pytest

import orc_tails as T
from test_parquet_footers_cpu import CODECS, KINDS, malformed, wide_file

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "orc")
PARQUET, ORC = 0, 1
PS_COMPRESSION, ZLIB, ZSTD = 2, 1, 5          # orc_proto PostScript.compression, CompressionKind


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = os.path.join(str(tmp_path_factory.mktemp("threads")), "threads_host_check")
    csrc = os.path.join(ROOT, "paimon_b200", "csrc")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-pthread", "-fsanitize=thread", "-I" + csrc, "-o", exe,
                           os.path.join(ROOT, "tests", "native", "threads_host_check.cc"),
                           os.path.join(csrc, "parquet_meta.cc"), os.path.join(csrc, "orc_meta.cc")])
    return exe


def run(exe, files):
    """files: [(PARQUET or ORC, bytes)] -> (exit status, stdout, stderr)"""
    inp = b"".join(struct.pack("<Bq", kind, len(b)) + b for kind, b in files)
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66 report_signal_unsafe=0")
    p = subprocess.run([exe], input=inp, capture_output=True, env=env)
    return p.returncode, p.stdout.decode(), p.stderr.decode(errors="replace")


def inputs():
    """Parquet files of every codec with many row groups; ORC files of every codec the reader takes, several stripes
    each, and the golden files; malformed files of both formats."""
    pq = [wide_file(seed, CODECS[seed % len(CODECS)], n=3000) for seed in range(6)]
    pq += [malformed(pq[i], kind) for i, kind in enumerate(KINDS)]
    orc = [open(os.path.join(GOLDEN, f), "rb").read() for f in sorted(os.listdir(GOLDEN)) if f.endswith(".orc")]
    for seed, codec in enumerate(["uncompressed", "zlib", "lz4", "zstd", "zlib", "zstd"]):
        orc.append(T.pyarrow_file(4000, seed=seed, compression=codec, stripe_size=4096, compression_block_size=65536))
    orc += list(T.malformed_tails().values())[:3]
    return [(PARQUET, b) for b in pq] + [(ORC, b) for b in orc]


@pytest.fixture(scope="module")
def files():
    return inputs()


def test_metadata_parses_on_eight_threads_equal_the_sequential_ones(driver, files):
    code, out, err = run(driver, files)
    assert "ThreadSanitizer" not in err, err[-6000:]
    assert code == 0, (code, out, err[-3000:])
    n = len(files)
    # 8 threads x 2 rounds: every file (shared), then the thread's own share of them (distinct)
    assert out.split() == ["files", str(n), "parses", str(2 * (8 * n + n)), "mismatches", "0"], out


def test_the_inputs_reach_every_path(files):
    """zlib and zstd ORC metadata (the per-thread inflate tables), multi-stripe tails, Parquet footers of every codec,
    and malformed files of both formats whose errors must be the same on every thread."""
    orc = [b for k, b in files if k == ORC][2:8]
    compression = {T.Tail.get(T.pb_fields(b[-1 - b[-1]:-1]), PS_COMPRESSION) for b in orc}
    assert {ZLIB, ZSTD} <= compression, compression
    assert len(T.Tail(T.pyarrow_file(6000, compression="uncompressed", stripe_size=4096)).stripes()) > 1
    assert sum(k == PARQUET for k, _ in files) == 6 + len(KINDS)
