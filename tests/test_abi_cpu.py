"""CPU-side checks of the C-ABI library: it loads, exports every symbol include/paimon_gpu.h declares,
validates handles, and refuses to run without a CUDA device (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

from paimon_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = set()
    for fn in os.listdir(os.path.join(ROOT, "include")):
        if fn.endswith(".h"):
            src = open(os.path.join(ROOT, "include", fn)).read()
            src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
            names |= set(re.findall(r"\b(pg_[a-z0-9_]+)\s*\(", src))
    return sorted(names)


def test_library_exports_every_declared_symbol():
    lib = N.load()
    decl = declared_symbols()
    assert len(decl) >= 15
    for name in decl:
        assert hasattr(lib, name), f"{name} declared in include/ but not exported"
    assert set(decl) == set(N.exported_symbols())
    assert lib.pg_abi_version() == 2


def test_no_cuda_device_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = N.load()
    st = lib.pg_init(0)
    assert st == 3 and b"no CPU fallback" in lib.pg_last_error()
    with pytest.raises(N.PaimonGpuError):
        N.init(0)


def test_handle_validation_without_device():
    lib = N.load()
    assert lib.pg_schema_free(12345) == 1
    assert lib.pg_merge_execute(999) == 1
    assert b"unknown" in lib.pg_last_error()

    # every handle kind (tag in the top byte: 1 schema ... 7 upload) refuses a handle it never issued
    n_rows = C.c_int64(0)
    entry_points = {
        1: [lambda h: lib.pg_schema_free(h), lambda h: lib.pg_schema_info(h, None, None)],
        2: [lambda h: lib.pg_merge_spec_free(h)],
        3: [lambda h: lib.pg_run_free(h), lambda h: lib.pg_run_layout(h, C.byref(n_rows), None, None, 0)],
        4: [lambda h: lib.pg_merge_free(h), lambda h: lib.pg_merge_stats(h, C.byref(N.PgStats()))],
        5: [lambda h: lib.pg_parquet_free(h), lambda h: lib.pg_parquet_describe(h, C.byref(N.PgParquetInfo()))],
        6: [lambda h: lib.pg_parquet_file_free(h), lambda h: lib.pg_parquet_file_meta(h, C.byref(N.PgFileMeta()))],
        7: [lambda h: lib.pg_files_upload_free(h), lambda h: lib.pg_files_upload_wait(h, None, 0)],
    }
    for tag, calls in entry_points.items():
        for call in calls:
            for h in (12345, (tag << 56) | 12345):
                assert call(h) == 1, (tag, h)
                assert b"unknown" in lib.pg_last_error(), (tag, h)

    # the kinds a host can create without a device carry their own tag, are refused by every other kind's free
    # function, and survive it
    import numpy as np
    import pyarrow as pa
    import pyarrow.parquet as pq
    field = N.PgField(4, 0)                                # PG_INT64
    desc = N.PgSchemaDesc(1, 0, C.pointer(field), None)
    schema, spec, reader = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    assert lib.pg_schema_create(C.byref(desc), C.byref(schema)) == 0
    assert lib.pg_merge_spec_create(schema.value, C.byref(N.PgMergeSpec()), C.byref(spec)) == 0
    sink = pa.BufferOutputStream()                         # [_KEY_k, _SEQUENCE_NUMBER, _VALUE_KIND], 3 rows
    pq.write_table(pa.table({"_KEY_k": pa.array([1, 2, 3], pa.int64()), "_SEQUENCE_NUMBER": pa.array([1, 2, 3], pa.int64()),
                             "_VALUE_KIND": pa.array([0, 0, 0], pa.int8())}),
                   sink, compression="none", use_dictionary=False, data_page_version="1.0")
    file_bytes = np.frombuffer(sink.getvalue().to_pybytes(), np.uint8)
    assert lib.pg_parquet_open(schema.value, file_bytes.ctypes.data, len(file_bytes), C.byref(reader)) == 0, \
        lib.pg_last_error()

    n_key, n_val = C.c_int32(-1), C.c_int32(-1)
    info = N.PgParquetInfo()
    frees = {1: lib.pg_schema_free, 2: lib.pg_merge_spec_free, 3: lib.pg_run_free, 4: lib.pg_merge_free,
             5: lib.pg_parquet_free, 6: lib.pg_parquet_file_free, 7: lib.pg_files_upload_free}
    live = [(1, schema.value, lambda: lib.pg_schema_info(schema.value, C.byref(n_key), C.byref(n_val)) == 0),
            (2, spec.value, None),
            (5, reader.value, lambda: lib.pg_parquet_describe(reader.value, C.byref(info)) == 0 and info.n_rows == 3)]
    for tag, h, alive in live:
        assert h >> 56 == tag
        for other, free in frees.items():
            if other == tag:
                continue
            assert free(h) == 1, (tag, other)
            assert b"unknown" in lib.pg_last_error()
            assert alive is None or alive(), (tag, other)
    assert (n_key.value, n_val.value) == (1, 0)
    for tag, h, _ in live:                                 # the schema first: the spec and the reader keep it alive
        assert frees[tag](h) == 0, tag
        assert frees[tag](h) == 1, tag                     # freed once
        assert b"unknown" in lib.pg_last_error(), tag
        if tag == 1:
            info = N.PgParquetInfo()
            assert lib.pg_parquet_describe(reader.value, C.byref(info)) == 0, lib.pg_last_error()
            assert (info.n_columns, info.n_rows) == (3, 3)


def test_bad_file_descriptors_are_refused_before_device_work():
    """A section read checks every file descriptor (memory kind, size, bytes, run index) before it touches the device,
    and an upload checks the same but for the run index."""
    lib = N.load()
    field = N.PgField(4, 0)                                # PG_INT64
    desc = N.PgSchemaDesc(1, 0, C.pointer(field), None)
    schema = C.c_uint64(0)
    assert lib.pg_schema_create(C.byref(desc), C.byref(schema)) == 0
    blob = (C.c_uint8 * 100)()
    bad = {"no bytes": N.PgFileDesc(None, 100, N.PG_MEM_HOST, 0),
           "negative size": N.PgFileDesc(C.addressof(blob), -1, N.PG_MEM_HOST, 0),
           "memory kind": N.PgFileDesc(C.addressof(blob), 100, 5, 0),
           "run index": N.PgFileDesc(C.addressof(blob), 100, N.PG_MEM_HOST, 1)}
    try:
        for case, d in bad.items():
            files = (N.PgFileDesc * 1)(d)
            runs = (C.c_uint64 * 1)()
            for read_section in (lib.pg_parquet_read_section, lib.pg_orc_read_section):
                assert read_section(schema.value, files, 1, 1, None, None, runs, None) == 1, case
                err = lib.pg_last_error()
                assert b"descriptor" in err or b"run index" in err, (case, err)
                assert b"pg_init" not in err, case
            if case != "run index":
                upload = C.c_uint64(0)
                assert lib.pg_files_upload_begin(files, 1, C.byref(upload)) == 1, case
                assert b"descriptor" in lib.pg_last_error() and b"pg_init" not in lib.pg_last_error(), case
    finally:
        assert lib.pg_schema_free(schema.value) == 0


def test_interval_partition_host_logic_matches_oracle():
    import random
    import numpy as np
    from oracle import pyoracle
    lib = N.load()
    rng = random.Random(5)
    for _ in range(200):
        n = rng.randrange(1, 40)
        mn = np.array([rng.randrange(0, 300) for _ in range(n)], np.int64)
        mx = mn + np.array([rng.randrange(0, 60) for _ in range(n)], np.int64)
        sec = np.zeros(n, np.int32)
        run = np.zeros(n, np.int32)
        ns = C.c_int32(0)
        assert lib.pg_interval_partition(n, mn.ctypes.data, mx.ctypes.data, sec.ctypes.data, run.ctypes.data,
                                         C.byref(ns)) == 0
        osec, orun, ons = pyoracle.interval_partition(mn.tolist(), mx.tolist())
        assert ns.value == ons
        assert sec.tolist() == osec.tolist()
        # run ids are labels: compare the partition into runs, not the labels
        def groups(s, r):
            g = {}
            for i, (a, b) in enumerate(zip(s.tolist(), r.tolist())):
                g.setdefault((a, b), []).append(i)
            return sorted(g.values())
        assert groups(sec, run) == groups(osec, orun)


def test_interval_partition_with_string_and_composite_key_bounds():
    """IntervalPartition over non-integer key bounds (strings compare as UTF-8 bytes, tuples field by field): the same
    sections / runs as over integer bounds with the same order."""
    import random
    from paimon_b200.merge_tree_readers import DataFileMeta, IntervalPartition
    rng = random.Random(9)
    for trial in range(20):
        n = rng.randrange(1, 30)
        bounds = []
        for _ in range(n):
            a, b = sorted((rng.randrange(100), rng.randrange(100)))
            bounds.append((a, b))
        def shape(files):
            return [[[f.file_name for f in run.files] for run in sec] for sec in IntervalPartition(files).partition()]
        ints = [DataFileMeta(f"f{i}", 0, 1, a, b) for i, (a, b) in enumerate(bounds)]
        strs = [DataFileMeta(f"f{i}", 0, 1, "k%03dé" % a, "k%03dé" % b) for i, (a, b) in enumerate(bounds)]
        tups = [DataFileMeta(f"f{i}", 0, 1, (a // 10, "x%d" % (a % 10)), (b // 10, "x%d" % (b % 10)))
                for i, (a, b) in enumerate(bounds)]
        assert shape(ints) == shape(strs) == shape(tups)


def test_jni_shim_binds_every_export_and_compiles():
    """jni/paimon_gpu_jni.cc calls every function include/paimon_gpu.h exports, and passes a syntax-only compile
    against the JNI specification's signatures (jni/stub/jni.h; the image has no JDK)."""
    import subprocess
    src = open(os.path.join(ROOT, "jni", "paimon_gpu_jni.cc")).read()
    code = re.sub(r"//[^\n]*", "", src)
    called = set(re.findall(r"\b(pg_[a-z0-9_]+)\s*\(", code))
    missing = [n for n in declared_symbols() if n not in called]
    assert not missing, f"exports without a JNI binding: {missing}"
    assert len(re.findall(r"JNIEXPORT", src)) >= 40
    res = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "jni", "stub"),
                          "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "jni", "paimon_gpu_jni.cc")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


def test_arrow_c_data_structs_match_pyarrow():
    """The ArrowSchema / ArrowArray definitions in include/paimon_gpu.h have the layout pyarrow's C interface uses."""
    from pyarrow.cffi import ffi
    assert ffi.sizeof("struct ArrowSchema") == 72 and ffi.sizeof("struct ArrowArray") == 80
    hdr = open(os.path.join(ROOT, "include", "paimon_gpu.h")).read()
    body = hdr[hdr.index("struct ArrowArray {"):]
    body = body[:body.index("};")]
    order = re.findall(r"(\w+)\s*(?:\)\s*\([^)]*\))?;", body)
    assert [n for n in order if n in ("length", "null_count", "offset", "n_buffers", "n_children", "buffers", "children",
                                      "dictionary", "release", "private_data")] == \
        ["length", "null_count", "offset", "n_buffers", "n_children", "buffers", "children", "dictionary", "release",
         "private_data"]
