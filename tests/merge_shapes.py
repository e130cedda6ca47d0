"""Seeded merge inputs built to reach the tile structures named in merge_tiles.py.

Every builder returns a Shape: host runs for the device merge and the oracle, the key ordinals the tile model
takes, and the structural edges (merge_tiles.edges) the shape claims to reach.  `scale` shrinks a shape for CPU
checks; the GPU tests use scale 1.  Sequence numbers are unique per key (ties are outside the reference's contract).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from paimon_b200.columnar import Column, KeyValueBatch, pack_validity
from paimon_b200.types import DataField, KeyValueSchema, PhysicalType, RowType

import merge_tiles as mt

P = PhysicalType


@dataclass
class Shape:
    name: str
    schema: KeyValueSchema
    runs: List[KeyValueBatch]
    ordinals: List[np.ndarray]
    rule: str = "all"
    start_rows: Optional[List[int]] = None
    lens_col: Optional[int] = None          # value column whose bytes the model counts per tile
    claims: set = field(default_factory=set)

    def plan(self) -> mt.TilePlan:
        seqs = [r.sequence_numbers for r in self.runs]
        kinds = [r.value_kinds for r in self.runs]
        lens = None
        if self.lens_col is not None:
            lens = []
            for r in self.runs:
                c = r.value_column(self.lens_col)
                ln = np.diff(np.asarray(c.offsets, np.int64))
                if c.valid is not None:
                    ln = ln * np.unpackbits(c.valid, bitorder="little")[: len(ln)]
                lens.append(ln)
        return mt.plan(self.ordinals, self.start_rows, seqs, kinds, self.rule, lens)


# ---- columns
def str_column(lens: np.ndarray, seed: int, valid: Optional[np.ndarray] = None, t=P.STRING) -> Column:
    """Strings of the given lengths, bytes from a seeded generator (printable)."""
    lens = np.asarray(lens, np.int64)
    offs = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    data = np.random.default_rng(seed).integers(0x21, 0x7f, int(offs[-1]), dtype=np.uint8)
    return Column(t, data, offs.astype(np.int32), None if valid is None else pack_validity(valid))


def bytes_column(values, t=P.STRING) -> Column:
    return Column.from_pylist(t, list(values))


def value_schema(key_fields, pk):
    """Key fields + v BIGINT, d DOUBLE, s STRING (all nullable)."""
    vt = RowType(tuple(key_fields) + (DataField("v", "BIGINT", True), DataField("d", "DOUBLE", True),
                                      DataField("s", "STRING", True)))
    return KeyValueSchema.of(vt, pk)


def run_batch(schema, key_cols, seq, kind, rng, null_prob=0.2, s_lens=None, s_valid=None) -> KeyValueBatch:
    """One run: the key columns, sequence numbers, kinds and seeded values for v, d and s."""
    n = len(seq)
    v_valid = rng.random(n) >= null_prob
    d_valid = rng.random(n) >= null_prob / 2
    if s_lens is None:
        s_lens = rng.integers(0, 13, n)
    if s_valid is None:
        s_valid = rng.random(n) >= null_prob
    vals = [Column(P.INT64, rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64), None, pack_validity(v_valid)),
            Column(P.DOUBLE, rng.uniform(-1e3, 1e3, n), None, pack_validity(d_valid)),
            str_column(s_lens, int(rng.integers(1 << 30)), s_valid)]
    return KeyValueBatch(schema, list(key_cols) + [Column(P.INT64, np.asarray(seq, np.int64)),
                                                   Column(P.INT8, np.asarray(kind, np.int8))] + list(key_cols) + vals)


def bigint_runs(name, keys_per_run, seqs, kinds=None, seed=0, claims=(), rule="all", **kw) -> Shape:
    schema = value_schema((DataField("k", "BIGINT", False),), ["k"])
    rng = np.random.default_rng(seed)
    runs = []
    for r, keys in enumerate(keys_per_run):
        kind = np.zeros(len(keys), np.int8) if kinds is None else kinds[r]
        runs.append(run_batch(schema, [Column(P.INT64, np.asarray(keys, np.int64))], seqs[r], kind, rng, **kw))
    return Shape(name, schema, runs, [np.asarray(k, np.int64) for k in keys_per_run], rule, claims=set(claims))


def unique_seqs(sizes, seed) -> List[np.ndarray]:
    """Globally unique sequence numbers in a random order across runs."""
    perm = np.random.default_rng(seed).permutation(int(sum(sizes))).astype(np.int64)
    return np.split(perm, np.cumsum(sizes)[:-1])


# ---- 1. full overlap: every key in every run
def full_overlap(k: int, n: int, seed: int = 1) -> Shape:
    keys = np.arange(n, dtype=np.int64) * 7 - n
    i = np.arange(n, dtype=np.int64)
    seqs = [i * k + (5 * r + i) % k for r in range(k)]        # a permutation of the runs per key (gcd(5, k) = 1)
    claims = {"odd_plan_tiles", "three_levels"} if (k, n) == (32, 20000) else set()
    return bigint_runs(f"full_overlap_k{k}_n{n}", [keys] * k, seqs, seed=seed, claims=claims)


FULL_OVERLAP = [(1, 1500), (2, 3000), (3, 40000), (17, 12000), (31, 1000), (32, 20000)]


# ---- 2. disjoint, interleaved and banded runs
def disjoint(k=8, m=40000, seed=2) -> Shape:
    keys = [np.arange(r * m, (r + 1) * m, dtype=np.int64) for r in range(k)]
    return bigint_runs("disjoint", keys, unique_seqs([m] * k, seed), seed=seed)


def interleaved(k=7, m=40000, seed=3) -> Shape:
    keys = [np.arange(m, dtype=np.int64) * k + r for r in range(k)]
    return bigint_runs("interleaved_mod_k", keys, unique_seqs([m] * k, seed), seed=seed)


def banded(k=6, m=40000, seed=4) -> Shape:
    keys = [np.arange(max(r * m - 1 - r % 3, 0), (r + 1) * m + 1 + r % 3, dtype=np.int64) for r in range(k)]
    return bigint_runs("banded_overlap", keys, unique_seqs([len(x) for x in keys], seed), seed=seed)


# ---- 3. skew
def skew(big=1_000_000, seed=5) -> Shape:
    rng = np.random.default_rng(seed)
    keys = [np.arange(big, dtype=np.int64) * 4 + 2]
    lo, hi, mid = 2, (big - 1) * 4 + 2, big * 2 + 2
    for r in range(31):
        cnt = r % 4
        anchor = (lo, hi, mid)[r % 3]
        cand = anchor + np.array([-1, 0, 1, 3], np.int64) * (1 + r // 3)
        keys.append(np.sort(rng.choice(cand, cnt, replace=False)))
    return bigint_runs("skew_one_big_run", keys, unique_seqs([len(x) for x in keys], seed), seed=seed)


def stride_lengths(seed=6) -> Shape:
    rng = np.random.default_rng(seed)
    sizes = [15, 16, 17, 255, 256, 257, 4095, 4096, 4097]
    keys = [np.sort(rng.choice(20000, n, replace=False)).astype(np.int64) for n in sizes]
    return bigint_runs("run_lengths_at_strides", keys, unique_seqs(sizes, seed), seed=seed)


# ---- 6. empty output
def delete_ranges(k=4, n=50000, block=3000, seed=7, rod=False) -> Shape:
    """Full overlap; every third block of `block` keys has only DELETE members (whole plan and emit tiles without
    output under drop-delete); elsewhere the newest member is a DELETE with probability 0.3."""
    rng = np.random.default_rng(seed)
    keys = np.arange(n, dtype=np.int64)
    i = keys
    seqs = [i * k + (3 * r + i) % k for r in range(k)]
    dead = (i // block) % 3 == 1
    kinds = []
    for r in range(k):
        kd = np.where(rng.random(n) < 0.3, 3, 0).astype(np.int8)
        kd[dead] = 3
        kinds.append(kd)
    return bigint_runs("delete_ranges_rod" if rod else "delete_ranges", [keys] * k, seqs, kinds, seed=seed,
                       rule="drop_delete", claims={"zero_row_emit_tile", "out_base_residues"})


def retract_only_groups(k=3, n=30000, seed=8) -> Shape:
    rng = np.random.default_rng(seed)
    keys = np.arange(n, dtype=np.int64) * 2
    i = np.arange(n)
    seqs = [i * k + (r + i) % k for r in range(k)]
    only = (i // 1500) % 4 == 2
    kinds = []
    for r in range(k):
        kd = rng.choice(np.array([0, 1, 2, 3], np.int8), n)
        kd[only] = rng.choice(np.array([1, 3], np.int8), int(only.sum()))
        kinds.append(kd)
    return bigint_runs("retract_only_groups", [keys] * k, seqs, kinds, seed=seed, rule="ignore_delete",
                       claims={"zero_row_emit_tile"})


def all_deleted(k=3, n=9000, seed=9) -> Shape:
    keys = np.arange(n, dtype=np.int64)
    seqs = [keys * k + r for r in range(k)]
    kinds = [np.full(n, 3, np.int8)] * k
    return bigint_runs("all_deleted", [keys] * k, seqs, kinds, seed=seed, rule="drop_delete")


# ---- 7. var-len look-back
def null_and_empty_ranges(k=3, n=60000, block=2500, seed=10) -> Shape:
    """String column s NULL (every fourth block) or "" (the block after) over whole tile ranges; elsewhere lengths
    cycle through 0..40."""
    rng = np.random.default_rng(seed)
    keys = np.arange(n, dtype=np.int64)
    i = keys
    seqs = [i * k + (r + i) % k for r in range(k)]
    b = (i // block) % 4
    lens = np.where(b == 2, 0, (i * 7 + 3) % 41)
    valid = b != 1
    sh = bigint_runs("null_and_empty_ranges", [keys] * k, seqs, seed=seed, s_lens=lens, s_valid=valid,
                     claims={"zero_byte_tile"})
    sh.lens_col = 3
    return sh


def one_huge_value(seed=11) -> Shape:
    n = 20000
    keys = np.arange(n, dtype=np.int64)
    seqs = [keys * 2, keys * 2 + 1]
    lens1 = (keys % 41).copy()
    lens1[n // 3] = 16 << 20
    schema = value_schema((DataField("k", "BIGINT", False),), ["k"])
    rng = np.random.default_rng(seed)
    runs = [run_batch(schema, [Column(P.INT64, keys)], seqs[0], np.zeros(n, np.int8), rng),
            run_batch(schema, [Column(P.INT64, keys)], seqs[1], np.zeros(n, np.int8), rng, s_lens=lens1,
                      s_valid=np.ones(n, bool))]
    return Shape("one_16MiB_value", schema, runs, [keys, keys])


# ---- 8. start rows
START_RESIDUES = [0, 1, 7, 8, 31, 32, 127]


def start_rows_shape(m=60000, seed=12) -> Shape:
    k = len(START_RESIDUES)
    keys = [np.sort(np.random.default_rng(seed + r).choice(3 * m, m, replace=False)).astype(np.int64)
            for r in range(k)]
    sh = bigint_runs("start_rows", keys, unique_seqs([m] * k, seed), seed=seed,
                     claims={"start_rows_strided"})
    sh.start_rows = list(START_RESIDUES)
    return sh


# ---- 5. non-exact keys across levels
def string_key_shape(name, key_lists, seed, t="STRING") -> Shape:
    """Runs of byte-string keys (each list sorted and unique)."""
    vt = RowType((DataField("k", t, False), DataField("v", "BIGINT", True), DataField("d", "DOUBLE", True),
                  DataField("s", "STRING", True)))
    schema = KeyValueSchema.of(vt, ["k"])
    ranks = mt.key_ranks([[(x,) for x in keys] for keys in key_lists])
    seqs = unique_seqs([len(x) for x in key_lists], seed)
    rng = np.random.default_rng(seed)
    pt = P.STRING if t == "STRING" else P.BINARY
    runs = [run_batch(schema, [bytes_column(keys, pt)], seqs[r], np.zeros(len(keys), np.int8), rng)
            for r, keys in enumerate(key_lists)]
    return Shape(name, schema, runs, ranks, claims={"three_levels"})


def changing_prefixes(k=4, m=160000, seed=13) -> Shape:
    """Keys share a prefix of more than 8 bytes inside a key range of 4000 keys, and the prefix changes from one
    range to the next; between the ranges sit prefix families "x", "x\\0", "x\\0\\0" spread over the runs."""
    total = k * m
    lists = [[] for _ in range(k)]
    for i in range(total):
        g = i // 4000
        base = b"tenant-%04d/region-%d/" % (g, g % 7)
        r = i % k
        if (i // 97) % 5 == 0:
            key = base + b"ab%06d" % (i // 3) + b"\0" * (i % 3)   # "x", "x\0", "x\0\0" in three different runs
        else:
            key = base + b"%08d" % i
        lists[r].append(key)
    return string_key_shape("changing_prefixes", [sorted(set(x)) for x in lists], seed)


def binary_high_bytes(k=4, m=160000, seed=14) -> Shape:
    rng = np.random.default_rng(seed)
    alphabet = np.array([0x00, 0x01, 0x7f, 0x80, 0xfe, 0xff], np.uint8)
    lists = []
    for r in range(k):
        s = set()
        while len(s) < m:
            ln = int(rng.integers(0, 11))
            s.add(bytes(alphabet[rng.integers(0, len(alphabet), ln)]))
        lists.append(sorted(s))
    return string_key_shape("binary_high_bytes", lists, seed, "BINARY")


def gpu_shapes() -> List:
    """(builder, kwargs) of every shape the GPU edge tests merge, with the edges each claims."""
    return ([(full_overlap, dict(k=k, n=n)) for k, n in FULL_OVERLAP] +
            [(disjoint, {}), (interleaved, {}), (banded, {}), (skew, {}), (stride_lengths, {}),
             (delete_ranges, {}), (delete_ranges, dict(rod=True)), (retract_only_groups, {}), (all_deleted, {}),
             (null_and_empty_ranges, {}), (one_huge_value, {}), (start_rows_shape, {}),
             (changing_prefixes, {}), (binary_high_bytes, {})])
