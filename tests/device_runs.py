"""Runs opened from device memory (pg_run_open with PG_MEM_DEVICE), in the buffer layouts the ABI allows, and the
bench's own device generator.

A host-opened run is copied into fresh 256-byte-aligned buffers; a device run reaches the kernels exactly as the caller
laid it out.  DeviceRun puts the bytes of a host KeyValueBatch into torch tensors in one of LAYOUTS:

  separate  one tensor per buffer, sized to the 16-byte round-up of its bytes and no more
  arena     every buffer of every column in one uint8 tensor at 16-byte-aligned offsets, none of them 256-byte
            aligned; the bytes between a buffer's end and its 16-byte round-up hold 0xFF
  aliased   the key column's buffers passed again for the value field of the same name (the bench does this)
  dirty     validity bits past n_rows set, extreme values (INT64 / INT32 min and max, NaN, +-inf) under fixed-width
            NULL slots, payload under var-len NULL cells
  based     var-len `data` at byte 0 of a longer payload whose first B bytes are 0xFF, absolute offsets from B > 0
            (B not a multiple of 16; 2^20 + 5 for the first var-len column when `big_base`)

DeviceRun.mirror() is the host batch the device holds, read back from the tensors with .cpu() (never through
pg_run_fetch); clean() of it is what the oracle takes.

gen_device_run, _splitmix64 and _hex_keys restate bench.py's generator (importing bench.py sets a process-wide cache
size); tests/test_bench_shapes_cpu.py holds them to bench.py's syntax trees.  bench_mirror() reads one generated run
back to the host the same way mirror() does."""
import numpy as np
import torch

from paimon_b200.columnar import Column, KeyValueBatch, pack_validity, unpack_validity
from paimon_b200.sort_merge_reader import DeviceColumn, SortedRunReader
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType, is_varlen, numpy_dtype

P = PhysicalType
LAYOUTS = ("separate", "arena", "aliased", "dirty", "based")
BIG_BASE = (1 << 20) + 5


def round16(n):
    return (n + 15) & ~15


def schema_all():
    """k BIGINT key; v BIGINT, d DOUBLE, s STRING, i INT, b BOOLEAN, y BINARY, g INT (all nullable)."""
    vt = RowType((DataField("k", "BIGINT", False), DataField("v", "BIGINT", True), DataField("d", "DOUBLE", True),
                  DataField("s", "STRING", True), DataField("i", "INT", True), DataField("b", "BOOLEAN", True),
                  DataField("y", "BINARY", True), DataField("g", "INT", True)))
    return KeyValueSchema.of(vt, ["k"])


def _strings(rng, n, valid, t, longest=24):
    lens = rng.integers(0, longest + 1, n) * valid
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    data = rng.integers(0x21, 0x7f, int(offs[-1]), dtype=np.uint8)
    return Column(t, data, offs.astype(np.int32), pack_validity(valid))


def model_run(schema, keys, seqs, kinds, seed, null_prob=0.3):
    """A host run of schema_all() with the given sorted keys, sequence numbers and kinds."""
    rng = np.random.default_rng(seed)
    n = len(keys)
    kc = Column(P.INT64, np.asarray(keys, np.int64))

    def valid():
        return rng.random(n) >= null_prob
    cols = [kc, Column(P.INT64, np.asarray(seqs, np.int64)), Column(P.INT8, np.asarray(kinds, np.int8)), kc,
            Column(P.INT64, rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64), None, pack_validity(valid())),
            Column(P.DOUBLE, rng.uniform(-1e3, 1e3, n), None, pack_validity(valid())),
            _strings(rng, n, valid(), P.STRING),
            Column(P.INT32, rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32), None, pack_validity(valid())),
            Column(P.BOOL, (rng.random(n) < 0.5).astype(np.uint8), None, pack_validity(valid())),
            _strings(rng, n, valid(), P.BINARY, 40),
            Column(P.INT32, rng.integers(0, 50, n).astype(np.int32), None, pack_validity(valid()))]
    return KeyValueBatch(schema, cols)


def model_runs(k, n, seed, delete_prob=0.0, key_space=None):
    """k runs of n rows each over a shared key space, with globally unique sequence numbers; a share `delete_prob`
    of the rows are retracts (UPDATE_BEFORE or DELETE)."""
    schema = schema_all()
    rng = np.random.default_rng(seed)
    key_space = key_space or max(2 * n, 1)
    keys = [np.sort(rng.choice(key_space, min(n, key_space), replace=False)).astype(np.int64) for _ in range(k)]
    perm = rng.permutation(sum(len(x) for x in keys)).astype(np.int64)
    seqs = np.split(perm, np.cumsum([len(x) for x in keys])[:-1])
    runs = []
    for r in range(k):
        kinds = np.where(rng.random(len(keys[r])) < delete_prob, rng.choice([1, 3], len(keys[r])), 0).astype(np.int8)
        runs.append(model_run(schema, keys[r], seqs[r], kinds, seed * 1000 + r))
    return runs


def clean(batch):
    """The batch with zeros under NULL slots, no payload under NULL cells, offsets from 0 and no validity bits
    past n_rows: what the run means, in the form the oracle takes."""
    return KeyValueBatch(batch.schema, [c if c is None or (c.valid is None and (c.offsets is None or c.offsets[0] == 0))
                                        else _canonical(c) for c in batch.columns])


def _canonical(c):
    out = c.canonical()
    return out if c.valid is not None else Column(out.type, out.data, out.offsets, None)


# ---------------------------------------------------------------------------------------------- layouts

_EXTREMES = {P.INT64: [-2 ** 63, 2 ** 63 - 1], P.INT32: [-2 ** 31, 2 ** 31 - 1],
             P.DOUBLE: [np.nan, np.inf, -np.inf, -0.0], P.FLOAT: [np.nan, np.inf, -np.inf], P.BOOL: [1, 0xFF],
             P.INT8: [-128, 127], P.INT16: [-2 ** 15, 2 ** 15 - 1]}


def _dirty_column(c, n):
    if c.valid is None:
        return c
    mask = unpack_validity(c.valid, n)
    vbytes = np.zeros((n + 7) // 8 + 8, np.uint8)
    vbytes[: (n + 7) // 8] = np.asarray(c.valid[: (n + 7) // 8], np.uint8)
    bits = np.unpackbits(vbytes, bitorder="little")
    bits[n:] = 1                                                  # every bit past the last row set
    vbytes = np.packbits(bits, bitorder="little")
    nulls = np.flatnonzero(~mask)
    if c.offsets is None:
        data = np.array(c.data[:n], copy=True)
        ext = np.array(_EXTREMES[P(c.type)], dtype=data.dtype)
        data[nulls] = ext[np.arange(len(nulls)) % len(ext)]
        return Column(c.type, data, None, vbytes)
    offs = np.asarray(c.offsets, np.int64)
    lens = np.diff(offs)
    lens[nulls] = 1 + nulls % 5                                   # payload under every NULL cell
    new = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=new[1:])
    data = np.full(int(new[-1]), ord("X"), np.uint8)
    rows = np.flatnonzero(mask)
    src_lens = np.diff(offs)[rows]
    within = np.arange(int(src_lens.sum())) - np.repeat(np.cumsum(src_lens) - src_lens, src_lens)
    data[np.repeat(new[rows], src_lens) + within] = np.asarray(c.data)[np.repeat(offs[rows], src_lens) + within]
    return Column(c.type, data, new.astype(np.int32), vbytes)


def _based_column(c, base):
    offs = np.asarray(c.offsets, np.int64)
    payload = np.asarray(c.data[int(offs[0]):int(offs[-1])], np.uint8)
    data = np.concatenate([np.full(base, 0xFF, np.uint8), payload])
    return Column(c.type, data, (offs - offs[0] + base).astype(np.int32), c.valid)


def layout_batch(batch, layout, big_base=False):
    """The host bytes a layout puts on the device (dirty and based change them; the others place them only)."""
    n = batch.n_rows
    if layout == "dirty":
        return KeyValueBatch(batch.schema, [_dirty_column(c, n) for c in batch.columns])
    if layout == "based":
        cols, j = [], 0
        for c in batch.columns:
            if c.offsets is not None:
                cols.append(_based_column(c, BIG_BASE if big_base and j == 0 else 13 + 48 * j))
                j += 1
            else:
                cols.append(c)
        return KeyValueBatch(batch.schema, cols)
    return batch


def _buffers(col, n):
    """(data, offsets, validity) host bytes of a column, as the ABI reads them."""
    t = P(col.type)
    if is_varlen(t):
        offs = np.ascontiguousarray(col.offsets[: n + 1], np.int32)
        data = np.ascontiguousarray(col.data[: int(offs[-1]) if n else 0], np.uint8)
    else:
        offs = None
        data = np.ascontiguousarray(col.data[:n], numpy_dtype(t))
    val = None if col.valid is None else np.ascontiguousarray(col.valid, np.uint8)
    return [data, offs, val]


class DeviceRun:
    """The bytes of `batch` (after layout_batch) in device tensors laid out as `layout`."""

    def __init__(self, batch, layout, big_base=False, device="cuda"):
        assert layout in LAYOUTS
        self.schema, self.layout, self.n_rows = batch.schema, layout, batch.n_rows
        host = layout_batch(batch, layout, big_base)
        n = self.n_rows
        names = [f.name for f in self.schema.file_fields()]
        nk = self.schema.n_key
        alias = {}
        if layout == "aliased":                                  # value field -> key column of the same name
            keys = {f.name[len("_KEY_"):]: i for i, f in enumerate(self.schema.key_type.fields)}
            alias = {nk + 2 + j: keys[f.name] for j, f in enumerate(self.schema.value_type.fields) if f.name in keys}
        self._types = self.schema.physical_types()
        bufs = [_buffers(c, n) for c in host.columns]
        self._spans = [[None, None, None] for _ in bufs]          # (tensor, byte offset, bytes) per buffer
        self.keep = []
        if layout == "arena":
            pos, places = 16, []
            for c, b in enumerate(bufs):
                for k, a in enumerate(b):
                    if a is None:
                        continue
                    if pos % 256 == 0:
                        pos += 16
                    places.append((c, k, pos, a))
                    pos += max(round16(a.nbytes), 16)
            arena = torch.full((pos + 256,), 0xFF, dtype=torch.uint8, device=device)
            shift = -arena.data_ptr() % 256                      # offsets are from a 256-byte boundary
            for c, k, off, a in places:
                off += shift
                if a.nbytes:
                    arena[off:off + a.nbytes] = torch.from_numpy(a.view(np.uint8).reshape(-1)).to(device)
                self._spans[c][k] = (arena, off, a.nbytes)
            self.keep.append(arena)
        else:
            for c, b in enumerate(bufs):
                if c in alias:
                    self._spans[c] = list(self._spans[alias[c]])
                    continue
                for k, a in enumerate(b):
                    if a is None:
                        continue
                    t = torch.full((max(round16(a.nbytes), 16),), 0xFF, dtype=torch.uint8, device=device)
                    if a.nbytes:
                        t[: a.nbytes] = torch.from_numpy(a.view(np.uint8).reshape(-1)).to(device)
                    self._spans[c][k] = (t, 0, a.nbytes)
                    self.keep.append(t)
        self.columns = [DeviceColumn(*[0 if s is None else s[0].data_ptr() + s[1] for s in sp]) for sp in self._spans]
        self.names = names

    def reader(self):
        return SortedRunReader.from_device(self.schema, self.n_rows, self.columns, keepalive=self)

    def mirror(self):
        """The batch the device buffers hold, read back with .cpu()."""
        cols = []
        for t, sp in zip(self._types, self._spans):
            raw = [None if s is None else s[0][s[1]:s[1] + s[2]].cpu().numpy() for s in sp]
            if is_varlen(t):
                cols.append(Column(t, raw[0], raw[1].view(np.int32), raw[2]))
            else:
                cols.append(Column(t, raw[0].view(numpy_dtype(t)), None, raw[2]))
        return KeyValueBatch(self.schema, cols)


# ---------------------------------------------------------------------------------------------- bench.py's generator

def _splitmix64(x):
    x = x + (-7046029254386353131)                       # 0x9E3779B97F4A7C15 as int64
    x = (x ^ ((x >> 30) & ((1 << 34) - 1))) * (-4658895280553007687)   # 0xBF58476D1CE4E5B9
    x = (x ^ ((x >> 27) & ((1 << 37) - 1))) * (-7723592293110705685)   # 0x94D049BB133111EB
    return x ^ ((x >> 31) & ((1 << 33) - 1))


def _hex_keys(keys, dev):
    """int64 keys -> 16-character lower-case hex strings (big endian: string order == integer order)."""
    import torch
    sh = torch.arange(60, -4, -4, device=dev, dtype=torch.int64)
    nib = ((keys[:, None] >> sh) & 15).to(torch.uint8)
    data = torch.where(nib < 10, nib + 48, nib + 87).flatten()
    data = torch.cat([data, torch.zeros(16, device=dev, dtype=torch.uint8)]).contiguous()
    offs = (torch.arange(keys.numel() + 1, device=dev, dtype=torch.int64) * 16).to(torch.int32).contiguous()
    return data, offs


def gen_device_run(schema, run_index, n, key_space, null_prob, seed, dev, delete_prob=0.0):
    """One sorted run generated directly in HBM.  Returns (columns, keepalive tensors, key tensor, bytes, kinds)."""
    import torch
    from paimon_b200.sort_merge_reader import DeviceColumn
    from paimon_b200.types import PhysicalType
    g = torch.Generator(device=dev)
    g.manual_seed(seed * 1000003 + run_index)
    keys = torch.randperm(key_space, device=dev, generator=g)[:n].sort().values.contiguous()
    keep = [keys]
    cols = []
    string_key = schema.key_type.fields[0].physical == PhysicalType.STRING
    if string_key:
        kdata, koffs = _hex_keys(keys, dev)
        keep += [kdata, koffs]
        key_col = DeviceColumn(kdata.data_ptr(), koffs.data_ptr())
        key_bytes = n * 16 + 4 * (n + 1)
    else:
        key_col = DeviceColumn(keys.data_ptr())
        key_bytes = n * 8
    for _ in schema.key_type.fields:
        cols.append(key_col)
    seq = (torch.arange(n, device=dev, dtype=torch.int64) + (run_index << 32)).contiguous()
    kind = torch.zeros(n, device=dev, dtype=torch.int8)
    if delete_prob > 0:
        kind[torch.rand(n, device=dev, generator=g) < delete_prob] = 3
    keep += [seq, kind]
    cols += [DeviceColumn(seq.data_ptr()), DeviceColumn(kind.data_ptr())]
    nbytes = key_bytes + seq.numel() * 8 + kind.numel()
    pk_names = {f.name[len("_KEY_"):] for f in schema.key_type.fields}
    for ci, f in enumerate(schema.value_type.fields):
        t = f.physical
        if f.name in pk_names:
            cols.append(key_col)
            nbytes += key_bytes
            continue
        h = _splitmix64(keys ^ ((run_index + 1) * 0x100 + ci << 40))
        valid_ptr = 0
        bits = None
        if f.nullable and null_prob > 0:
            assert null_prob == 0.5, "device generator draws validity bits with p = 0.5"
            vbytes = torch.randint(0, 256, ((n + 7) // 8 + 8,), device=dev, dtype=torch.uint8, generator=g)
            keep.append(vbytes)
            valid_ptr = vbytes.data_ptr()
            nbytes += (n + 7) // 8
            if t in (PhysicalType.STRING, PhysicalType.BINARY):
                sh = torch.arange(8, device=dev, dtype=torch.uint8)
                bits = ((vbytes[:, None] >> sh) & 1).flatten()[:n].to(torch.int64)
        if t == PhysicalType.INT64:
            keep.append(h)
            cols.append(DeviceColumn(h.data_ptr(), 0, valid_ptr))
            nbytes += n * 8
        elif t == PhysicalType.INT32:
            v = (h & 0x7fffffff).to(torch.int32).contiguous()
            keep.append(v)
            cols.append(DeviceColumn(v.data_ptr(), 0, valid_ptr))
            nbytes += n * 4
        elif t == PhysicalType.DOUBLE:
            d = ((h >> 11) & ((1 << 53) - 1)).to(torch.float64) * (2000.0 / (1 << 53)) - 1000.0
            keep.append(d)
            cols.append(DeviceColumn(d.data_ptr(), 0, valid_ptr))
            nbytes += n * 8
        elif t in (PhysicalType.STRING, PhysicalType.BINARY):
            lens = 8 + ((h >> 3) & 0xffff) % 17                       # U[8, 24]
            if bits is not None:
                lens = lens * bits                                     # NULL cells carry no payload
            offs = torch.zeros(n + 1, device=dev, dtype=torch.int64)
            torch.cumsum(lens, 0, out=offs[1:])
            total = int(offs[-1].item())
            offs32 = offs.to(torch.int32)
            data = torch.randint(48, 112, (max(total, 1) + 16,), device=dev, dtype=torch.uint8, generator=g)
            keep += [offs32, data]
            cols.append(DeviceColumn(data.data_ptr(), offs32.data_ptr(), valid_ptr))
            nbytes += total + 4 * (n + 1)
            del lens, offs, bits
        else:
            raise ValueError(f"bench generator: unsupported type {t}")
    return cols, keep, keys, nbytes, kind


def bench_mirror(schema, n, cols, keep):
    """The host batch of one gen_device_run run, read from its tensors with .cpu(): every column pointer is the
    start of one of the kept tensors."""
    by_ptr = {t.data_ptr(): t for t in keep}

    def raw(ptr, nbytes):
        return by_ptr[ptr].cpu().numpy().view(np.uint8)[:nbytes]
    out = []
    for t, dc in zip(schema.physical_types(), cols):
        valid = raw(dc.validity, (n + 7) // 8).copy() if dc.validity else None
        if is_varlen(t):
            offs = raw(dc.offsets, 4 * (n + 1)).view(np.int32).copy()
            out.append(Column(t, raw(dc.data, int(offs[-1])).copy(), offs, valid))
        else:
            w = np.dtype(numpy_dtype(t)).itemsize
            out.append(Column(t, raw(dc.data, n * w).view(numpy_dtype(t)).copy(), None, valid))
    return KeyValueBatch(schema, out)
