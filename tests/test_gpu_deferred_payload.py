"""Section decodes whose var-len columns take the deferred payload path: the value walk and the main-stream expansion
are enqueued before the host reads the payload sizes back, and the PLAIN BYTE_ARRAY expansion follows on the side
stream once the payload buffers exist.  PLAIN strings, dictionary strings, a projection that reads a single string
column and a section whose strings are all NULL decode to what pyarrow reads from the same bytes.  A page that the
levels pass refuses makes that read-back report an error while the other expansions are already enqueued: the
section is refused with PG_ERR_FORMAT, and the next decode on the same thread is correct."""
import io
import struct

import numpy as np
import pyarrow.parquet as pq
import pytest

import parquet_pages as P
from paimon_b200 import _native as N
from paimon_b200 import datagen
from paimon_b200.columnar import KeyValueBatch
from paimon_b200.format import read_section
from paimon_b200.merge_tree_readers import concat_batches
from paimon_b200.types import DataField, KeyValueSchema, RowType

from parquet_util import arrow_to_batch, write_kv_parquet

pytestmark = pytest.mark.gpu

PG_ERR_FORMAT = 6
SCHEMA = datagen.schema_c3(n_i64=2, n_f64=1, n_str=3)


def _fetch_and_close(readers):
    out = []
    for r in readers:
        try:
            out.append(r.read_batch())
        finally:
            r.close()
    return out


def _section(tmp_path, schema, run_sizes, opts, null_prob=0.3, str_len=(0, 120)):
    """Files written by pyarrow, several per run -> (files, per-run batches as pyarrow reads them)."""
    files, want, key0, fi = [], [], 0, 0
    for r, sizes in enumerate(run_sizes):
        parts = []
        for n in sizes:
            keys = np.arange(key0, key0 + 3 * n, 3, dtype=np.int64)
            key0 += 3 * n + 7
            part = datagen.make_run(schema, fi, keys, seed=11 + fi, null_prob=null_prob, str_len=str_len)
            path = str(tmp_path / f"f{fi}.parquet")
            write_kv_parquet(part, path, **opts[fi % len(opts)])
            files.append((open(path, "rb").read(), r))
            parts.append(arrow_to_batch(schema, pq.read_table(path)))
            fi += 1
        want.append(concat_batches(schema, parts))
    return files, want


def _check_runs(got, want):
    for r, (g, w) in enumerate(zip(got, want)):
        assert g.equals(w), f"run {r}: " + g.first_difference(w)


RUNS = [[3001, 1237], [64, 20_000], [4099]]


def test_plain_strings(tmp_path):
    opts = [dict(use_dictionary=False), dict(use_dictionary=False, data_page_version="2.0", data_page_size=4096),
            dict(use_dictionary=False, compression="zstd", data_page_size=1024)]
    files, want = _section(tmp_path, SCHEMA, RUNS, opts)
    readers, info = read_section(SCHEMA, files, len(RUNS))
    _check_runs(_fetch_and_close(readers), want)
    assert info.n_dictionary_pages == 0


def test_dictionary_strings(tmp_path):
    opts = [dict(), dict(data_page_version="2.0", compression="snappy"), dict(dictionary_pagesize_limit=1024)]
    files, want = _section(tmp_path, SCHEMA, RUNS, opts, str_len=(0, 12))
    readers, info = read_section(SCHEMA, files, len(RUNS))
    _check_runs(_fetch_and_close(readers), want)
    assert info.n_dictionary_pages > 0


@pytest.mark.parametrize("dictionary", [False, True])
def test_projection_of_a_single_string_column(tmp_path, dictionary):
    files, want = _section(tmp_path, SCHEMA, RUNS, [dict(use_dictionary=dictionary)])
    mask = [n == "s1" for n in SCHEMA.value_type.field_names()]
    assert sum(mask) == 1
    readers, _ = read_section(SCHEMA, files, len(RUNS), read_value_fields=mask)
    _check_runs(_fetch_and_close(readers), [w.project(mask) for w in want])


def test_all_null_strings(tmp_path):
    schema = KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("s", "STRING", True),
                                        DataField("b", "BINARY", True))), ["pk"])
    files = []
    for i, n in enumerate((5000, 33, 20_000)):
        batch = KeyValueBatch.from_rows(schema, [(k, k, 0, k, None, None) for k in range(i * 100_000, i * 100_000 + n)])
        path = str(tmp_path / f"n{i}.parquet")
        write_kv_parquet(batch, path, use_dictionary=i == 1)
        files.append((open(path, "rb").read(), i))
    readers, _ = read_section(schema, files, 3)
    got = _fetch_and_close(readers)
    for (blob, _), g in zip(files, got):
        w = arrow_to_batch(schema, pq.read_table(io.BytesIO(blob)))
        assert g.equals(w), g.first_difference(w)


def _levels_file(n, refused):
    """A KeyValue file [pk, v INT (OPTIONAL), s STRING (OPTIONAL, PLAIN)].  refused: the definition-level length of
    v's page points far past its body, so the levels pass marks the page bad."""
    valid = [k % 5 != 0 for k in range(n)]
    vals = [k * 7 for k in range(n) if valid[k]]
    strs = [b"s%d" % k for k in range(n) if valid[k]]
    if refused:
        v_page = P.data_page_v1(n, struct.pack("<I", 1 << 20) + P.plain(P.INT32, vals), P.E_PLAIN)
    else:
        v_page = P.data_page_v1(n, P.plain(P.INT32, vals), P.E_PLAIN, defs=P.levels(valid))
    s_page = P.data_page_v1(n, P.plain(P.BYTE_ARRAY, strs), P.E_PLAIN, defs=P.levels(valid))
    cols = [P.ValueColumn("v", P.INT32, True, [[v_page]]), P.ValueColumn("s", P.BYTE_ARRAY, True, [[s_page]],
                                                                           converted=P.UTF8)]
    return P.kv_file([n], cols)


def test_page_refused_by_the_levels_pass_with_expansions_enqueued(tmp_path):
    schema = KeyValueSchema.of(RowType((DataField("pk", "BIGINT", False), DataField("v", "INT", True),
                                        DataField("s", "STRING", True))), ["pk"])
    good = _levels_file(3000, False)
    bad = _levels_file(3000, True)
    plain_files, want = _section(tmp_path, SCHEMA, [[20_000]], [dict(use_dictionary=False)])
    with pytest.raises(N.PaimonGpuError) as ei:
        readers, _ = read_section(schema, [(good, 0), (bad, 1), (good, 2)], 3)
        _fetch_and_close(readers)
    assert ei.value.status == PG_ERR_FORMAT

    # the next decodes on this thread: the same layout without the bad page, then a section of another schema
    readers, _ = read_section(schema, [(good, 0), (good, 1)], 2)
    for g in _fetch_and_close(readers):
        w = arrow_to_batch(schema, pq.read_table(io.BytesIO(good)))
        assert g.equals(w), g.first_difference(w)
    readers, _ = read_section(SCHEMA, plain_files, 1)
    _check_runs(_fetch_and_close(readers), want)
