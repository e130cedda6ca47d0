"""Builds tests/native/codec_host_check.cc, the host build of the page decompressors, under AddressSanitizer and UBSan,
and runs records through it.  The decoders run in a child process, so the sanitizer runtime need not be preloaded into
Python, and every buffer is allocated at its exact size."""
import os
import struct
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LZ4_RAW, LZ4_HADOOP = 5, 6            # the filter's LZ4 modes, after codec_corpora's SNAPPY .. ZLIB = 0 .. 4


def build(tmp_dir: str):
    """-> run(records): records of (mode, src bytes, cap) -> [(result, output bytes)]"""
    exe = os.path.join(tmp_dir, "codec_host_check")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I" + os.path.join(ROOT, "paimon_b200", "csrc"), "-o", exe,
                           os.path.join(ROOT, "tests", "native", "codec_host_check.cc")])

    def run(records):
        inp = b"".join(struct.pack("<Bqq", m, cap, len(src)) + bytes(src) for m, src, cap in records)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        p = subprocess.run([exe], input=inp, capture_output=True, env=env)
        assert p.returncode == 0, p.stderr.decode(errors="replace")[-3000:]
        out, pos = [], 0
        for _ in records:
            (r,) = struct.unpack_from("<q", p.stdout, pos)
            pos += 8
            out.append((r, p.stdout[pos:pos + max(r, 0)]))
            pos += max(r, 0)
        assert pos == len(p.stdout)
        return out
    return run
