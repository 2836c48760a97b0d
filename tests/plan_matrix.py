"""The tuning options of a plain context, a pairwise covering array over them, and the reference result of
an evaluation on any of the plans they select -- TEST INFRASTRUCTURE ONLY.

No option may change a result (include/b200dpf.h), so every row of ``pairwise_rows`` must give ``expected``
bit for bit.  ``expected`` never comes from a GPU run:

  * standard keys: the host evaluation's shares (``eval_cpu``) times the table, with the shares of the first
    two keys checked against the C oracle's tree expansion (``Oracle.eval_full``) and a shard's partial of the
    first key against the oracle's (``Oracle.eval_dot_shard``) -- the oracle alone costs about 0.5 s per AES
    key at n = 2^16;
  * early-terminated keys: the host evaluation's shares (``eval_cpu_et``) times the table, with the shares of
    the first two keys checked against per-index walks (tests/et_oracle.py);
  * XOR-shared keys: the XOR of the rows whose host share bit (``eval_cpu_xor``) is set, with the bits of the
    first two keys checked against per-index walks (tests/xor_oracle.py);
  * a ``Sparse`` table (n >= 2^20): per-index walks over its support only (tests/sparse_oracle.py) for standard
    and early-terminated keys; for XOR-shared keys the host bits of the support rows, those of at most four
    keys checked leaf by leaf against ``xor_oracle.leaf_value``.

A shard's partial is restricted to the rows that shard owns: natural row i of a table of 2^lane_bits rows per
leaf belongs to shard r of G iff ((i >> lane_bits) & (G - 1)) == bitrev_g(r).
"""
import itertools
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import et_oracle  # noqa: E402
import sparse_oracle  # noqa: E402
import xor_oracle  # noqa: E402

# every option of b200dpf_ctx_set_option on a plain context, its default first, then the levels the matrix
# takes: both ends of each range, and the sizes the planner treats differently in between
OPTIONS = {
    "one_launch": (1, 0),
    "frontier": (1, 0),
    "frontier_mb": (256, 1),
    "subtree_log2": (0, 1, 3, 16),
    "top_log2": (0, 1, 3, 7),
    "balance_top": (1, 0),
    "lane_split": (1, 0),
    "leaf_cache": (1, 0),
    "leaf_cache_mb": (16384, 1),
    "mac_tma": (1, 0),
    "tma_rows": (0, 1),
    "timing": (0, 1),
}
DEFAULTS = {name: levels[0] for name, levels in OPTIONS.items()}

KINDS = ("standard", "et", "xor")
LANE_BITS = {"standard": 0, "et": 2, "xor": 7}
N_MIN = {"standard": 2, "et": 8, "xor": 256}


def _uncovered():
    names = list(OPTIONS)
    return {((a, va), (b, vb)) for a, b in itertools.combinations(names, 2)
            for va in OPTIONS[a] for vb in OPTIONS[b]}


def _pairs_of(row):
    names = list(OPTIONS)
    return {((a, row[a]), (b, row[b])) for a, b in itertools.combinations(names, 2)}


def pairwise_rows(seed=0, candidates=24):
    """Rows (dicts option -> level) such that every pair of levels of every two options is in one of them;
    the first row is all defaults.  Greedy: each row is the best of `candidates` rows, each built around one
    uncovered pair by giving every other option, in a random order, the level that covers most uncovered
    pairs with the options already set.  Deterministic for a seed."""
    rng = random.Random(seed)
    names = list(OPTIONS)
    left = _uncovered()
    rows = [dict(DEFAULTS)]
    left -= _pairs_of(rows[0])
    while left:
        best, best_gain = None, -1
        pool = sorted(left)
        for _ in range(candidates):
            (a, va), (b, vb) = pool[rng.randrange(len(pool))]
            row = {a: va, b: vb}
            for name in rng.sample([x for x in names if x not in row], len(names) - 2):
                def gain(v):
                    return sum(((f, row[f]), (name, v)) in left if names.index(f) < names.index(name)
                               else ((name, v), (f, row[f])) in left for f in row)
                levels = list(OPTIONS[name])
                rng.shuffle(levels)
                row[name] = max(levels, key=gain)
            row = {x: row[x] for x in names}
            g = len(_pairs_of(row) & left)
            if g > best_gain:
                best, best_gain = row, g
        rows.append(best)
        left -= _pairs_of(best)
    return rows


class Sparse:
    """An n x e table that is zero except on the rows of `units` (indices, or leaves of 2^lane_bits rows):
    every key of a batch is checked exactly from per-index walks over the support alone."""

    def __init__(self, kind, n, e, targets, shard_counts=(), seed=0):
        self.kind, self.n, self.e = kind, n, e
        self.rpl = 1 << LANE_BITS[kind]
        depth = n.bit_length() - 1 - LANE_BITS[kind]
        targets = np.asarray(targets, np.int64) >> LANE_BITS[kind]
        self.units = sparse_oracle.support(depth, targets, self.rpl, shard_counts, seed)
        self.rows = sparse_oracle.rows_of(self.units, self.rpl)
        self.vals = sparse_oracle.values(len(self.rows), e, seed + 1)

    def table(self):
        return sparse_oracle.host_table(self.n, self.rows, self.vals)

    @property
    def shape(self):
        return (self.n, self.e)

    def __getitem__(self, idx):
        """rows of the table (alphas drawn from the support)"""
        idx = np.asarray(idx, np.int64)
        pos = np.searchsorted(self.rows, idx)
        pos = np.minimum(pos, len(self.rows) - 1)
        out = np.zeros((len(idx), self.e), np.int32)
        hit = self.rows[pos] == idx
        out[hit] = self.vals[pos[hit]]
        return out


_ORC = None


def oracle():
    global _ORC
    if _ORC is None:
        import oracle as O
        _ORC = O.Oracle()
    return _ORC


def owned_rows(kind, n, shard_rank, shard_count):
    """mask over the n natural rows of the rows shard (shard_rank, shard_count) holds"""
    g = shard_count.bit_length() - 1
    return ((np.arange(n, dtype=np.int64) >> LANE_BITS[kind]) & (shard_count - 1)) == int(sparse_oracle.bitrev(shard_rank, g))


_CHECKED = set()     # (prf, key bytes) whose host shares were checked against per-index walks


def _unchecked(keys, prf, count):
    """indices of the first `count` keys not checked yet (a shape's keys are checked once, not once per shard)"""
    todo = []
    for k in range(min(count, len(keys))):
        tag = (prf, keys[k].tobytes())
        if tag not in _CHECKED:
            _CHECKED.add(tag)
            todo.append(k)
    return todo


def _check_et_shares(keys, prf, shares):
    """the host shares of up to two keys against per-index walks, on both ends and a sample of leaves"""
    leaves = shares.shape[1] // 4
    rng = np.random.RandomState(leaves)
    sample = np.unique(np.concatenate([[0, leaves - 1], rng.randint(0, leaves, size=min(leaves, 30))]))
    for k in _unchecked(keys, prf, 2):
        for j in sample:
            want = np.array(et_oracle.eval_flat_et(oracle(), keys[k], int(j), prf), np.uint32)
            assert np.array_equal(shares[k, 4 * j:4 * j + 4].view(np.uint32), want), (k, j)


def _check_xor_bits(keys, prf, words, leaves, nkeys):
    """host share bits (uint32 words over the whole table) of up to `nkeys` keys against xor_oracle.leaf_value
    on `leaves`"""
    for k in _unchecked(keys, prf, nkeys):
        for j in leaves:
            v = xor_oracle.leaf_value(oracle(), keys[k], int(j), prf)
            got = words[k, 4 * j:4 * j + 4].astype(object)
            assert int(got[0]) | int(got[1]) << 32 | int(got[2]) << 64 | int(got[3]) << 96 == v, (k, j)


def _xor_words(keys, prf):
    import b200dpf as B
    return np.stack([B.eval_cpu_xor(k, prf) for k in keys])


def expected(kind, prf, keys, table, shard_rank=0, shard_count=1):
    """int32 [len(keys), E]: the result of evaluating `keys` of `kind` on `table` (an int32 [n, E] array or a
    Sparse), or on its shard (shard_rank, shard_count)"""
    import b200dpf as B
    keys = np.ascontiguousarray(keys, np.int32).reshape(-1, 524)
    orc = oracle()
    if isinstance(table, Sparse):
        sp = table
        mask = sparse_oracle.owned(sp.units, shard_rank, shard_count) if shard_count > 1 else None
        if kind != "xor":
            return sparse_oracle.reference(orc, keys, prf, sp.units, sp.vals, sp.rpl, mask)
        words = _xor_words(keys, prf)
        _check_xor_bits(keys, prf, words, sp.units, 4)
        rows, vals = sp.rows, sp.vals
        if mask is not None:
            keep = np.repeat(mask, sp.rpl)
            rows, vals = rows[keep], vals[keep]
        bits = ((words[:, rows >> 5] >> (rows & 31).astype(np.uint32)) & 1).astype(np.uint8)
        return xor_oracle.xor_rows(bits, vals)
    table = np.ascontiguousarray(table, np.int32)
    n = table.shape[0]
    own = owned_rows(kind, n, shard_rank, shard_count) if shard_count > 1 else slice(None)
    if kind == "standard":
        shares = np.stack([B.eval_cpu(k, prf) for k in keys])
        for k in _unchecked(keys, prf, 2):
            assert np.array_equal(shares[k], orc.eval_full(keys[k], prf)), k
        out = et_oracle.dot_u32(shares[:, own], table[own])
        if shard_count > 1:     # the shard's rows by its range of tree positions, from the oracle alone
            pos = n // shard_count
            assert np.array_equal(out[0], orc.eval_dot_shard(keys[0], prf, table, shard_rank * pos, pos))
        return out
    if kind == "et":
        shares = np.stack([B.eval_cpu_et(k, prf) for k in keys])
        _check_et_shares(keys, prf, shares)
        return et_oracle.dot_u32(shares[:, own], table[own])
    words = _xor_words(keys, prf)
    leaves = n >> 7
    _check_xor_bits(keys, prf, words, range(leaves) if leaves <= 512 else
                    np.unique(np.random.RandomState(leaves).randint(0, leaves, 256)), 2)
    bits = np.stack([xor_oracle.unpack_bits(w) for w in words])
    return xor_oracle.xor_rows(bits[:, own], table[own])


def expected_shares(kind, prf, keys):
    """what b200dpf_expand_device writes for `keys`: int32 [B, n] shares (standard, early-terminated) or
    uint32 [B, n / 32] packed share bits (XOR-shared), natural row order"""
    import b200dpf as B
    if kind == "standard":
        return np.stack([oracle().eval_full(k, prf) for k in keys])
    if kind == "et":
        return np.stack([B.eval_cpu_et(k, prf) for k in keys])
    return _xor_words(keys, prf)


def combine(kind, parts):
    """the whole-table result from the shards' partials: their sum mod 2^32, or XOR"""
    acc = np.zeros_like(parts[0], dtype=np.uint32)
    for p in parts:
        acc = acc ^ p.view(np.uint32) if kind == "xor" else acc + p.view(np.uint32)
    return acc.view(np.int32)


def reconstruct(kind, ra, rb):
    a, b = np.asarray(ra, np.int32).view(np.uint32), np.asarray(rb, np.int32).view(np.uint32)
    return (a ^ b if kind == "xor" else a - b).view(np.int32)


def gen_keys(kind, n, alphas, prf, seed=0):
    import b200dpf as B
    gen = {"standard": B.gen_batch_secure, "et": B.gen_batch_et, "xor": B.gen_batch_xor}[kind]
    seeds = np.random.RandomState(seed).randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
    return gen(np.asarray(alphas, np.int64), n, seeds, prf)
