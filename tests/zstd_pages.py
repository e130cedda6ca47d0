"""PLAIN data page V1 bodies (definition levels + values, as the compaction output encoder lays them out) of the
lineitem-shaped C5 columns and of the C3 datagen shape, for the zstd encoder tests.  Built on the host with numpy from
the same generators bench.py and paimon_b200.datagen use, so the ratio checks see the bytes the device compresses."""
import numpy as np


def _def_prefix(n_rows: int, valid: np.ndarray) -> bytes:
    """[length:int32][bit-packed run header varint][validity bitmap bytes], bit width 1."""
    groups = (n_rows + 7) // 8
    v = (groups << 1) | 1
    hdr = bytearray()
    while v >= 0x80:
        hdr.append((v & 0x7F) | 0x80)
        v >>= 7
    hdr.append(v)
    bits = np.packbits(valid.astype(np.uint8), bitorder="little").tobytes()
    return (len(hdr) + groups).to_bytes(4, "little") + bytes(hdr) + bits


def plain_body(values, valid=None, optional=True) -> bytes:
    """One page body: `values` a numpy array (fixed width) or a list of bytes (BYTE_ARRAY)."""
    n = len(values)
    if valid is None:
        valid = np.ones(n, bool)
    out = _def_prefix(n, valid) if optional else b""
    if isinstance(values, np.ndarray):
        vals = values[valid]
        if vals.dtype in (np.int8, np.int16):
            vals = vals.astype(np.int32)
        return out + vals.tobytes()
    return out + b"".join(len(s).to_bytes(4, "little") + s for s, ok in zip(values, valid) if ok)


def c5_pages(n_rows=100_000, page_rows=20_000, seed=5):
    """Page bodies of every column of a C5 run (bench.c5_bucket's generators, key columns REQUIRED)."""
    rng = np.random.default_rng(seed)
    idx = np.arange(n_rows, dtype=np.int64)
    ok, ln = idx // 4, (idx % 4 + 1).astype(np.int32)
    flags = [np.array([b"A", b"N", b"R"]), np.array([b"F", b"O"])]
    instr = np.array([b"DELIVER IN PERSON", b"COLLECT COD", b"NONE", b"TAKE BACK RETURN"])
    modes = np.array([b"REG AIR", b"AIR", b"RAIL", b"SHIP", b"TRUCK", b"MAIL", b"FOB"])
    ship = rng.integers(8000, 10600, n_rows).astype(np.int32)
    cols = [(ok, False), (ln, False), (np.arange(n_rows, dtype=np.int64), False), (np.zeros(n_rows, np.int8), False),
            (ok, True), (ln, True), (rng.integers(1, 20_000_000, n_rows), True), (rng.integers(1, 1_000_000, n_rows), True)]
    cols += [(rng.integers(100, 5_000_000, n_rows), True) for _ in range(4)]
    cols += [(list(flags[0][rng.integers(0, 3, n_rows)]), True), (list(flags[1][rng.integers(0, 2, n_rows)]), True)]
    cols += [(ship, True), (ship + 30, True), (ship + 45, True)]
    cols += [(list(instr[rng.integers(0, 4, n_rows)]), True), (list(modes[rng.integers(0, 7, n_rows)]), True)]
    a, b = rng.integers(0, 1 << 40, n_rows), rng.integers(0, 1 << 30, n_rows)
    cols.append(([b"%d carefully final %d" % (x, y) for x, y in zip(a, b)], True))
    pages = []
    for vals, optional in cols:
        for p0 in range(0, n_rows, page_rows):
            pages.append(plain_body(vals[p0:p0 + page_rows], optional=optional))
    return pages


def c3_pages(n_rows=60_000, page_rows=20_000, seed=3):
    """Page bodies of the C3 datagen shape (int64 / float64 / string values, half of them NULL)."""
    rng = np.random.default_rng(seed)
    pages = []
    keys = np.sort(rng.choice(10 * n_rows, n_rows, replace=False)).astype(np.int64)
    cols = [(keys, None, False), (np.arange(n_rows, dtype=np.int64), None, False)]
    for _ in range(3):
        cols.append((rng.integers(-(1 << 40), 1 << 40, n_rows), rng.random(n_rows) >= 0.5, True))
    for _ in range(2):
        cols.append((rng.normal(size=n_rows), rng.random(n_rows) >= 0.5, True))
    for _ in range(2):
        cols.append(([b"v%d" % x for x in rng.integers(0, 1 << 30, n_rows)], rng.random(n_rows) >= 0.5, True))
    for vals, valid, optional in cols:
        for p0 in range(0, n_rows, page_rows):
            pages.append(plain_body(vals[p0:p0 + page_rows], None if valid is None else valid[p0:p0 + page_rows],
                                    optional))
    return pages
