"""The sparse-table oracle (tests/sparse_oracle.py) and keys at every depth up to n = 2^31, without a
GPU.  The oracle is what checks the GPU at large n (tests/test_gpu_large_domain.py), so here it is
checked itself: against the dense oracles at small n, and against corrupted share vectors that stand
for the ways a kernel goes wrong (a skipped or doubled range of positions, a wrong bit reversal)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402
import et_oracle  # noqa: E402
import sparse_oracle as S  # noqa: E402

PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)


def std_keys(n, batch, prf, seed):
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=batch).astype(np.int64)
    a, b = B.gen_batch_secure(alphas, n, rng.randint(0, 256, size=44 * batch).astype(np.uint8).tobytes(), prf)
    return a, b, alphas


def et_keys(n, batch, prf, seed):
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=batch).astype(np.int64)
    a, b = B.gen_batch_et(alphas, n, rng.randint(0, 256, size=44 * batch).astype(np.uint8).tobytes(), prf)
    return a, b, alphas


def to_positions(natural, depth, rows_per_leaf=1):
    """share vector in natural row order -> [position][rows_per_leaf] order"""
    v = natural.reshape(-1, rows_per_leaf)
    return v[S.bitrev(np.arange(1 << depth), depth)]


def to_natural(by_pos, depth):
    out = np.empty_like(by_pos)
    out[S.bitrev(np.arange(1 << depth), depth)] = by_pos
    return out.reshape(-1)


# ---- the sparse reference equals the dense oracles --------------------------------------------------

@pytest.mark.parametrize("prf", PRFS)
def test_sparse_reference_equals_dense_oracle(oracle, prf):
    n, e, depth = 1 << 13, 5, 13
    a, b, alphas = std_keys(n, 6, prf, seed=prf)
    units = S.support(depth, alphas, shard_counts=(4,), seed=1)
    assert len(units) < n                  # a real subset: 4096 blocks of two positions, plus marks
    vals = S.values(len(units), e, seed=2)
    table = S.host_table(n, units, vals)
    for keys in (a, b):
        want = oracle.eval_dot(keys, prf, table)
        assert np.array_equal(S.reference(oracle, keys, prf, units, vals), want)
    # shards: the ownership rule picks each shard's positions, and the partials add up
    parts = []
    for r in range(4):
        got = S.reference(oracle, a, prf, units, vals, mask=S.owned(units, r, 4))
        for k in range(2):
            assert np.array_equal(got[k], oracle.eval_dot_shard(a[k], prf, table, r * n // 4, n // 4))
        parts.append(got.view(np.uint32))
    assert np.array_equal(np.sum(parts, axis=0, dtype=np.uint32).view(np.int32), oracle.eval_dot(a, prf, table))
    rec = S.sub_u32(S.reference(oracle, a, prf, units, vals), S.reference(oracle, b, prf, units, vals))
    assert np.array_equal(rec, table[alphas])


@pytest.mark.parametrize("prf", PRFS)
def test_sparse_reference_equals_dense_oracle_et(oracle, prf):
    n, e = 1 << 10, 3
    depth = 8
    a, b, alphas = et_keys(n, 3, prf, seed=10 + prf)
    leaves = S.support(depth, alphas >> 2, rows_per_leaf=4, shard_counts=(2,), seed=3)
    rows = S.rows_of(leaves, 4)
    vals = S.values(len(rows), e, seed=4)
    table = S.host_table(n, rows, vals)
    want_a = et_oracle.eval_dot_et(oracle, a, prf, table)
    assert np.array_equal(S.reference(oracle, a, prf, leaves, vals, rows_per_leaf=4), want_a)
    # the C walk equals the Python restatement leaf by leaf
    pts = oracle.eval_points_et(a[:1], prf, leaves[:40])
    assert np.array_equal(pts[0].view(np.uint32), np.array([et_oracle.eval_flat_et(oracle, a[0], int(v), prf) for v in leaves[:40]], np.uint32).reshape(-1))
    parts = [S.reference(oracle, a, prf, leaves, vals, 4, S.owned(leaves, r, 2)).view(np.uint32) for r in range(2)]
    assert np.array_equal(np.sum(parts, axis=0, dtype=np.uint32).view(np.int32), want_a)
    rec = S.sub_u32(want_a, S.reference(oracle, b, prf, leaves, vals, rows_per_leaf=4))
    assert np.array_equal(rec, table[alphas])


def test_support_covers_every_block_and_mark():
    depth = 31
    alphas = np.array([0, 5, (1 << 31) - 1], np.int64)
    units = S.support(depth, alphas, shard_counts=(4,))
    pos = S.bitrev(units, depth)
    blk = (1 << depth) // S.BLOCKS
    assert np.array_equal(np.unique(pos // blk), np.arange(S.BLOCKS))
    for m in [0, (1 << 31) - 1] + [k * (1 << 26) + d for k in range(1, 32) for d in (-1, 0)] + [1 << 30, (1 << 29) - 1]:
        assert m in set(pos.tolist()), m
    for a in alphas:
        assert {int(a), int(a) ^ (1 << 30), int(a) ^ 1} <= set(units.tolist())
    # early-terminated: leaf positions, row marks divided by four
    leaves = S.support(29, alphas >> 2, rows_per_leaf=4, shard_counts=(4,))
    lpos = set(S.bitrev(leaves, 29).tolist())
    assert {(1 << 24) - 1, 1 << 24, (1 << 28) - 1, 1 << 28, (1 << 27) - 1} <= lpos


# ---- the sparse check catches what it claims ----------------------------------------------------------

def _corruptions(by_pos, depth):
    """share vectors in position order, corrupted the ways a traversal goes wrong"""
    npos = 1 << depth
    blk = npos // S.BLOCKS if npos >= S.BLOCKS else 1
    k = 3 * (npos // blk) // 5
    out = {}
    z = by_pos.copy()
    z[k * blk:(k + 1) * blk] = 0                       # one block of positions skipped
    out["skipped block"] = z
    d = by_pos.copy()
    d[(k + 1) * blk:(k + 2) * blk] = by_pos[k * blk:(k + 1) * blk]   # a block written twice
    out["doubled block"] = d
    out["first position skipped"] = np.concatenate([np.zeros_like(by_pos[:1]), by_pos[1:]])
    out["last position skipped"] = np.concatenate([by_pos[:-1], np.zeros_like(by_pos[:1])])
    # bit reversal off by one level: position p treated as holding rotl(bitrev(p), 1)
    p = np.arange(npos)
    rot = ((S.bitrev(p, depth) << 1) | (S.bitrev(p, depth) >> (depth - 1))) & (npos - 1)
    shifted = np.empty_like(by_pos)
    shifted[S.bitrev(rot, depth)] = by_pos
    out["bit reversal shifted"] = shifted
    return out


@pytest.mark.parametrize("prf", (B.PRF_CHACHA20, B.PRF_AES128))
def test_sparse_check_catches_corrupted_shares(oracle, prf):
    n, depth, e = 1 << 14, 14, 2
    a, _, alphas = std_keys(n, 2, prf, seed=20 + prf)
    units = S.support(depth, alphas, seed=5)
    vals = S.values(len(units), e, seed=6)
    table = S.host_table(n, units, vals)
    want = S.reference(oracle, a, prf, units, vals)
    for k in range(2):
        natural = oracle.eval_full(a[k], prf)
        assert np.array_equal(S.dot_u32(natural[None, :], table), want[k:k + 1])
        for what, bad in _corruptions(to_positions(natural, depth, 1), depth).items():
            got = S.dot_u32(to_natural(bad, depth)[None, :], table)
            assert not np.array_equal(got, want[k:k + 1]), "sparse check missed: " + what


def test_sparse_check_catches_corrupted_shares_et(oracle):
    prf, n, e = B.PRF_SALSA20, 1 << 14, 2
    depth = 12
    a, _, alphas = et_keys(n, 1, prf, seed=30)
    leaves = S.support(depth, alphas >> 2, rows_per_leaf=4, seed=7)
    rows = S.rows_of(leaves, 4)
    vals = S.values(len(rows), e, seed=8)
    table = S.host_table(n, rows, vals)
    want = S.reference(oracle, a, prf, leaves, vals, rows_per_leaf=4)
    natural = oracle.eval_points_et(a, prf, np.arange(n // 4))[0]
    assert np.array_equal(S.dot_u32(natural[None, :], table), want)
    for what, bad in _corruptions(to_positions(natural, depth, 4), depth).items():
        got = S.dot_u32(to_natural(bad, depth)[None, :], table)
        assert not np.array_equal(got, want), "sparse check missed: " + what


# ---- keys at every depth ------------------------------------------------------------------------------

def _probe_indices(alpha, depth, rng):
    """alpha, alpha with each single bit flipped, and random indices"""
    n = 1 << depth
    idx = [alpha] + [alpha ^ (1 << j) for j in range(depth)] + list(rng.randint(0, n, size=8))
    return np.array(idx, np.int64)


def _check_point_function(oracle, ka, kb, prf, alpha, depth, rng):
    idx = _probe_indices(alpha, depth, rng)
    d = S.sub_u32(oracle.eval_points(ka, prf, idx), oracle.eval_points(kb, prf, idx))[0]
    assert np.array_equal(d, (idx == alpha).astype(np.int32)), (depth, prf, alpha)


@pytest.mark.parametrize("prf", PRFS)
def test_keys_at_every_depth(oracle, prf):
    rng = np.random.RandomState(40 + prf)
    for depth in range(1, 32):
        n = 1 << depth
        alpha = int(rng.randint(0, n))
        seed = rng.randint(0, 256, size=44).astype(np.uint8).tobytes()
        for ka, kb in (B.gen(alpha, n, int(rng.randint(0, 2**31)), prf), B.gen_secure(alpha, n, seed, prf)):
            assert B.lib().b200dpf_key_depth(ka) == depth and B.lib().b200dpf_key_n(ka) == n
            _check_point_function(oracle, ka, kb, prf, alpha, depth, rng)
        alphas = np.array([0, n - 1, alpha], np.int64)
        seeds = rng.randint(0, 256, size=44 * 3).astype(np.uint8).tobytes()
        ka, kb = B.gen_batch_secure(alphas, n, seeds, prf)
        for k, al in enumerate(alphas):
            _check_point_function(oracle, ka[k], kb[k], prf, int(al), depth, rng)
            # the batch is the single-key generator, key by key
            sa, sb = B.gen_secure(int(al), n, seeds[44 * k:44 * (k + 1)], prf)
            assert np.array_equal(sa, ka[k]) and np.array_equal(sb, kb[k])


@pytest.mark.parametrize("prf", PRFS)
def test_et_keys_at_every_depth(oracle, prf):
    rng = np.random.RandomState(50 + prf)
    for logn in range(3, 32):
        n, depth = 1 << logn, logn - 2
        for alpha in (0, n - 1, int(rng.randint(0, n))):
            ka, kb = B.gen_et(alpha, n, rng.randint(0, 256, size=44).astype(np.uint8).tobytes(), prf)
            assert et_oracle.key_depth(ka) == depth
            leaf = alpha >> 2
            leaves = np.array([leaf] + [leaf ^ (1 << j) for j in range(depth)] + list(rng.randint(0, n // 4, size=6)), np.int64)
            d = S.sub_u32(oracle.eval_points_et(ka, prf, leaves), oracle.eval_points_et(kb, prf, leaves))[0]
            want = (S.rows_of(leaves, 4) == alpha).astype(np.int32)
            assert np.array_equal(d, want), (logn, prf, alpha)


def test_compact_keys_at_depth_31():
    n, alpha = 1 << 31, (1 << 31) - 3
    ka, kb = B.gen_secure(alpha, n, bytes(range(44)), B.PRF_AES128)
    for k in (ka, kb):
        packed = B.key_pack(k)
        assert len(packed) == 2016 == B.lib().b200dpf_key_packed_size(31)
        assert np.array_equal(B.key_unpack(packed), k)
    ea, eb = B.gen_et(alpha, n, bytes(range(44)), B.PRF_AES128)
    for k in (ea, eb):
        packed = B.key_pack_et(k)
        assert len(packed) == B.lib().b200dpf_key_packed_size(29) == 32 + 64 * 29
        assert np.array_equal(B.key_unpack_et(packed), k)


# ---- the per-index walk against the reference at depths the golden files never reach ----------------

@pytest.mark.parametrize("prf", PRFS)
def test_eval_flat_matches_reference_at_depths_25_to_30(oracle, ref, prf):
    rng = np.random.RandomState(60 + prf)
    for depth in range(25, 31):
        n = 1 << depth
        alpha = int(rng.randint(0, n))
        seed = int(rng.randint(0, 2**31))
        ka, kb = ref.gen(alpha, n, seed, prf)
        oa, ob = oracle.gen(alpha, n, seed, prf)
        assert np.array_equal(ka, oa) and np.array_equal(kb, ob)
        idx = _probe_indices(alpha, depth, rng)[:12]
        for key in (ka, kb):
            for i in idx:
                assert oracle.eval_flat(key, int(i), prf) == ref.eval_flat(key, int(i), prf), (depth, int(i))
