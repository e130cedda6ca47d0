"""Write KeyValue batches as Paimon-shaped Parquet data files with pyarrow (the byte-level decode oracle,
SURVEY.md §8c): file schema [_KEY_*, _SEQUENCE_NUMBER BIGINT NOT NULL, _VALUE_KIND TINYINT NOT NULL, value...]."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from paimon_b200.columnar import Column, KeyValueBatch, pack_validity, unpack_validity
from paimon_b200.types import PhysicalType, is_varlen, numpy_dtype

_PA = {PhysicalType.INT8: pa.int8(), PhysicalType.INT16: pa.int16(), PhysicalType.INT32: pa.int32(),
       PhysicalType.INT64: pa.int64(), PhysicalType.FLOAT: pa.float32(), PhysicalType.DOUBLE: pa.float64(),
       PhysicalType.STRING: pa.string(), PhysicalType.BINARY: pa.binary(), PhysicalType.BOOL: pa.bool_()}


def to_arrow(batch: KeyValueBatch) -> pa.Table:
    fields, arrays = [], []
    for f, col in zip(batch.schema.file_fields(), batch.columns):
        t = f.physical
        n = len(col)
        mask = None if col.valid is None else ~unpack_validity(col.valid, n)
        if is_varlen(t):
            vals = col.to_pylist()
            arr = pa.array(vals, type=_PA[t])
        else:
            data = np.asarray(col.data[:n])
            if t == PhysicalType.BOOL:
                data = data.astype(bool)
            arr = pa.array(data, type=_PA[t], mask=mask)
        fields.append(pa.field(f.name, _PA[t], nullable=f.nullable))
        arrays.append(arr)
    return pa.Table.from_arrays(arrays, schema=pa.schema(fields))


def write_kv_parquet(batch: KeyValueBatch, path: str, **kw) -> None:
    opts = dict(compression="none", use_dictionary=True, data_page_version="1.0", write_statistics=False)
    opts.update(kw)
    pq.write_table(to_arrow(batch), path, **opts)


def arrow_to_column(t: PhysicalType, arr: pa.Array) -> Column:
    """One pyarrow array as the Column Column.from_pylist(t, arr.to_pylist()) builds: validity None without NULLs,
    zeros under NULL slots, var-len payload without bytes under NULL slots.  Integer, floating, boolean, string and
    binary arrays are taken from their buffers (the tests compare files of millions of rows); other arrow types go
    through Python values."""
    n = len(arr)
    mask = None if arr.null_count == 0 else np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), bool)
    valid = None if mask is None else pack_validity(mask)
    at = arr.type
    if n and is_varlen(t) and (pa.types.is_string(at) or pa.types.is_binary(at)):
        bufs = arr.buffers()
        offs = np.frombuffer(bufs[1], np.int32)[arr.offset:arr.offset + n + 1].astype(np.int64)
        data = np.frombuffer(bufs[2], np.uint8) if bufs[2] is not None else np.zeros(0, np.uint8)
        lens = np.diff(offs)
        if mask is not None and lens[~mask].any():                 # payload under a NULL slot: drop it
            keep = np.repeat(mask, lens)
            data = data[offs[0]:offs[-1]][keep]
            lens = lens * mask
            new = np.zeros(n + 1, np.int64)
            np.cumsum(lens, out=new[1:])
            return Column(t, data.copy(), new.astype(np.int32), valid)
        return Column(t, data[offs[0]:offs[-1]].copy(), (offs - offs[0]).astype(np.int32), valid)
    if not is_varlen(t) and (pa.types.is_integer(at) or pa.types.is_floating(at) or pa.types.is_boolean(at)):
        vals = arr.fill_null(False if pa.types.is_boolean(at) else 0).to_numpy(zero_copy_only=False)
        return Column(t, np.asarray(vals).astype(numpy_dtype(t)), None, valid)
    return Column.from_pylist(t, arr.to_pylist())


def arrow_to_batch(schema, table: pa.Table) -> KeyValueBatch:
    cols = []
    for f, name in zip(schema.file_fields(), table.column_names):
        cols.append(arrow_to_column(f.physical, table.column(name).combine_chunks()))
    return KeyValueBatch(schema, cols)
