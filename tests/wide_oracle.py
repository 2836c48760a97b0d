"""Exact reference results for entries of up to 4096 columns -- TEST INFRASTRUCTURE ONLY.

``common.dot_u32`` loops over columns in Python, which takes seconds per shape at 4096 columns.
``dot_u32_exact`` gets the same bits from three float64 matrix products: with every uint32 written as
lo + 2^16 * hi (16-bit limbs),

    sum_i s_i * t_i  mod 2^32  =  sum s_lo * t_lo  +  2^16 * ((sum s_lo * t_hi + sum s_hi * t_lo) mod 2^16)   mod 2^32.

Every limb product is below 2^32, so over at most 2^20 rows every partial sum is an integer below 2^52 and
float64 holds it exactly, whatever order the matrix product adds in.  Rows go in chunks of at most 2^20 (each
reduced in integers), columns in chunks that bound the host memory.

``expected`` is the result of evaluating keys of a kind on a table (or a shard of it), from the host
evaluation's shares, with the shares of the first two keys of each (kind, prf, keys) checked against the
independent per-index oracles as tests/plan_matrix.py does: ``Oracle.eval_full`` (standard), per-leaf walks of
tests/et_oracle.py (early-terminated) and ``xor_oracle.leaf_value`` (XOR-shared).  XOR-shared results are
``xor_oracle.xor_rows``.  References are cached by (kind, prf, keys, table, shard).
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import plan_matrix as PM  # noqa: E402
import xor_oracle  # noqa: E402

ROW_CHUNK = 1 << 20      # the most rows whose limb-product sums stay below 2^52
COL_CHUNK = 512


def dot_u32_exact(shares, table, row_chunk=ROW_CHUNK, col_chunk=COL_CHUNK):
    """int32 share vectors [B, n] (or [n]) x int32 table [n, E] -> int32 [B, E], wrapping mod 2^32"""
    if not 1 <= row_chunk <= ROW_CHUNK or col_chunk < 1:
        raise ValueError("row_chunk must be in [1, 2^20] and col_chunk positive")
    s = np.atleast_2d(np.asarray(shares, np.int32)).view(np.uint32)
    t = np.asarray(table, np.int32).view(np.uint32)
    if t.ndim != 2 or s.shape[1] != t.shape[0]:
        raise ValueError("shares [B, n] and table [n, E] do not match: %s, %s" % (s.shape, t.shape))
    acc = np.zeros((s.shape[0], t.shape[1]), np.uint64)
    for r0 in range(0, t.shape[0], row_chunk):
        sc = s[:, r0:r0 + row_chunk]
        s_lo, s_hi = (sc & 0xFFFF).astype(np.float64), (sc >> 16).astype(np.float64)
        for c0 in range(0, t.shape[1], col_chunk):
            tc = t[r0:r0 + row_chunk, c0:c0 + col_chunk]
            t_lo, t_hi = (tc & 0xFFFF).astype(np.float64), (tc >> 16).astype(np.float64)
            low = (s_lo @ t_lo).astype(np.uint64)
            mid = (s_lo @ t_hi).astype(np.uint64) + (s_hi @ t_lo).astype(np.uint64)
            acc[:, c0:c0 + col_chunk] = (acc[:, c0:c0 + col_chunk] + low + ((mid & 0xFFFF) << 16)) & 0xFFFFFFFF
    return acc.astype(np.uint32).view(np.int32)


def _digest(a):
    a = np.ascontiguousarray(a)
    return (a.shape, hashlib.blake2b(a.view(np.uint8), digest_size=16).digest())


_CACHE = {}


def expected(kind, prf, keys, table, shard_rank=0, shard_count=1):
    """int32 [len(keys), E]: the result of evaluating `keys` of `kind` on the int32 [n, E] `table`, or on its
    shard (shard_rank, shard_count)"""
    import b200dpf as B
    keys = np.ascontiguousarray(keys, np.int32).reshape(-1, 524)
    table = np.ascontiguousarray(table, np.int32)
    tag = (kind, prf, _digest(keys), _digest(table), shard_rank, shard_count)
    if tag in _CACHE:
        return _CACHE[tag]
    n = table.shape[0]
    own = PM.owned_rows(kind, n, shard_rank, shard_count) if shard_count > 1 else slice(None)
    if kind == "standard":
        shares = np.stack([B.eval_cpu(k, prf) for k in keys])
        for k in PM._unchecked(keys, prf, 2):
            assert np.array_equal(shares[k], PM.oracle().eval_full(keys[k], prf)), k
        out = dot_u32_exact(shares[:, own], table[own])
    elif kind == "et":
        shares = np.stack([B.eval_cpu_et(k, prf) for k in keys])
        PM._check_et_shares(keys, prf, shares)
        out = dot_u32_exact(shares[:, own], table[own])
    else:
        words = PM._xor_words(keys, prf)
        leaves = n >> 7
        PM._check_xor_bits(keys, prf, words, range(leaves) if leaves <= 512 else
                           np.unique(np.random.RandomState(leaves).randint(0, leaves, 256)), 2)
        bits = np.stack([xor_oracle.unpack_bits(w) for w in words])
        out = xor_oracle.xor_rows(bits[:, own], table[own])
    _CACHE[tag] = out
    return out


def clear_cache():
    _CACHE.clear()
