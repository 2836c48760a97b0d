"""Sparse-table oracle for large domains -- TEST INFRASTRUCTURE ONLY.

A table that is zero except on a support S gives the exact result from |S| per-index walks:

    out[b][e] = sum_{i in S} low32(EvaluateFlat(key_b, i)) * T[i][e]   (mod 2^32)

Each share comes from its own root-to-leaf walk in the C oracle (``Oracle.eval_points`` /
``eval_points_et``), which shares nothing with the engine's traversal (no bit-reversed positions,
work items, frontier, shards or leaf cache).  A check costs O(|S| * depth) per key, so every key of a
batch can be compared bit-exactly at any n.

S is chosen in POSITION space, where the engine's structure lives: position p of a tree of depth d
holds unit bitrev_d(p), where a unit is a natural index for standard keys and a leaf (rows 4*leaf ..
4*leaf + 3) for early-terminated ones.  A device table is stored in position order, so a skipped,
doubled or misplaced range of positions is a range of table rows.  ``support`` takes

  * one random position in every aligned block of P/4096 positions (P = 2^d), so any skipped or
    doubled range that long changes the result;
  * positions 0 and P-1, and those just before and after every multiple of 2^26 and 2^30 table rows
    (a 64-byte row at 2^26 starts at 4 GiB) and of every shard boundary;
  * for each key's target unit a: a, its sibling a ^ (1 << (d-1)) (the last bit a walk consumes, so
    they share a parent: positions p and p ^ 1) and a ^ 1 (the first bit: the other half of the tree).
"""
import numpy as np

BLOCKS = 4096
ROW_MARKS = (1 << 26, 1 << 30)      # table rows whose 64-byte row starts at 4 GiB and at 64 GiB


def bitrev(x, bits):
    """bit reversal of the low `bits` bits, elementwise over an int64 array"""
    x = np.asarray(x, np.int64)
    r = np.zeros_like(x)
    for k in range(bits):
        r |= ((x >> k) & 1) << (bits - 1 - k)
    return r


def support(depth, targets, rows_per_leaf=1, shard_counts=(), seed=0):
    """Sorted unique units (indices, or leaves when rows_per_leaf = 4) of a tree of `depth` levels;
    `targets`: each key's target unit (alpha, or alpha >> 2 for early-terminated keys)."""
    npos = 1 << depth
    rng = np.random.RandomState(seed)
    nblocks = min(BLOCKS, npos)
    blk = npos // nblocks
    pos = [np.arange(nblocks, dtype=np.int64) * blk + rng.randint(0, blk, size=nblocks)]
    marks = [0, npos - 1]
    for m in [r // rows_per_leaf for r in ROW_MARKS] + [npos // g for g in shard_counts if g > 1]:
        for k in range(m, npos, m):
            marks += [k - 1, k]
    pos.append(np.array(marks, np.int64))
    units = [bitrev(np.concatenate(pos), depth)]
    t = np.asarray(targets, np.int64).reshape(-1)
    if depth >= 1:
        units += [t, t ^ (1 << (depth - 1)), t ^ 1]
    return np.unique(np.concatenate(units))


def rows_of(units, rows_per_leaf=1):
    """table rows of the units, in unit order (a leaf's four rows together)"""
    u = np.asarray(units, np.int64)
    if rows_per_leaf == 1:
        return u
    return (u[:, None] * rows_per_leaf + np.arange(rows_per_leaf)).reshape(-1)


def owned(units, shard_rank, shard_count):
    """mask of the units shard (shard_rank, shard_count) owns (include/b200dpf.h): natural index i iff
    (i & (G-1)) == bitrev_g(rank), and for early-terminated keys leaf v = i >> 2 iff (v & (G-1)) ==
    bitrev_g(rank) -- the same rule on units.  Its positions are [rank * P/G, (rank+1) * P/G)."""
    g = shard_count.bit_length() - 1
    return (np.asarray(units, np.int64) & (shard_count - 1)) == int(bitrev(shard_rank, g))


def values(nrows, entry_size, seed):
    """full-range random int32 rows for the support"""
    return np.random.RandomState(seed).randint(-2**31, 2**31, size=(nrows, entry_size), dtype=np.int64).astype(np.int32)


def host_table(n, rows, vals):
    """int32 [n, E] zero except vals at rows.  np.zeros leaves the untouched pages unallocated."""
    t = np.zeros((n, vals.shape[1]), np.int32)
    t[rows] = vals
    return t


def shares(orc, keys, prf, units, rows_per_leaf=1):
    """int32 [B, len(rows_of(units))]: each key's share of each support row, by per-index walks"""
    if rows_per_leaf == 1:
        return orc.eval_points(keys, prf, units)
    return orc.eval_points_et(keys, prf, units)


def dot_u32(s, t):
    """int32 [B, m] x int32 [m, E] -> int32 [B, E] mod 2^32 (exact: products reduced before summing)"""
    s = np.asarray(s, np.int32).view(np.uint32).astype(np.uint64)
    t = np.asarray(t, np.int32).view(np.uint32).astype(np.uint64)
    out = np.zeros((s.shape[0], t.shape[1]), np.uint64)
    for e in range(t.shape[1]):
        out[:, e] = ((s * t[:, e][None, :]) & np.uint64(0xFFFFFFFF)).sum(axis=1) & np.uint64(0xFFFFFFFF)
    return out.astype(np.uint32).view(np.int32)


def reference(orc, keys, prf, units, vals, rows_per_leaf=1, mask=None):
    """the exact result on a table that is `vals` at rows_of(units) and zero elsewhere; `mask` (over
    units) restricts the sum to one shard's units"""
    units = np.asarray(units, np.int64)
    if mask is not None:
        keep = np.repeat(mask, rows_per_leaf)
        units, vals = units[mask], vals[keep]
    return dot_u32(shares(orc, keys, prf, units, rows_per_leaf), vals)


def sub_u32(a, b):
    return (np.asarray(a, np.int32).view(np.uint32) - np.asarray(b, np.int32).view(np.uint32)).view(np.int32)
