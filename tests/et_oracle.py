"""Per-index oracle for early-terminated DPF keys -- TEST INFRASTRUCTURE ONLY.

These functions restate the definition of early-terminated keys (DESIGN.md section 9) and share no
code with the engine's tree walk: every leaf is reached by its own root-to-leaf walk, one PRF call
per level, through the pinned PRF of the C oracle (oracle/dpf_oracle.c, ``orc_prf``).  The
reference has no such keys, so nothing here is pinned against it; what pins the construction is
that both servers' shares reconstruct the one-hot row vector, and the golden file
tests/golden/et_v1.npz.

    leaf j = i >> 2, lane l = i & 3, tree depth d = log2(n) - 2
    step k = 0 .. d-1 consumes bit k of j (the root takes the least significant bit) with
    correction-word level L = d-1-k, bank cw_2 when the parent seed is odd, else cw_1:
        child = PRF(parent, bit) + cw[2L + bit]        mod 2^128, for L > 0
        child = PRF(parent, bit) + cw[2L + bit]        lane-wise in (Z/2^32)^4, for L = 0
    share[i] = lane l of the leaf value
"""
import numpy as np

KEY_WORDS = 524
M128 = (1 << 128) - 1


def _slot(key, s):
    w = np.asarray(key, np.int32).view(np.uint32)[4 * s:4 * s + 4]
    return int(w[0]) | int(w[1]) << 32 | int(w[2]) << 64 | int(w[3]) << 96


def _lanes(v):
    return [(v >> (32 * l)) & 0xFFFFFFFF for l in range(4)]


def key_depth(key):
    """tree depth d of an early-terminated key (slot 0 = (d, 2, 0, 0)), n = 4 * 2^d rows"""
    k = np.asarray(key, np.int32)
    assert int(k[1]) == 2 and int(k[2]) == 0 and int(k[3]) == 0, "not an early-terminated key"
    d = int(k[0])
    assert _slot(k, 130) == 4 << d
    return d


def eval_flat_et(orc, key, leaf, prf):
    """the four 32-bit words of leaf `leaf` (rows 4*leaf .. 4*leaf+3)"""
    d = key_depth(key)
    seed = _slot(key, 129)
    for k in range(d):
        bit = (leaf >> k) & 1
        level = d - 1 - k
        cw = _slot(key, (65 if seed & 1 else 1) + 2 * level + bit)
        v = orc.prf(prf, seed, bit)
        if level > 0:
            seed = (v + cw) & M128
        else:
            seed = sum(((a + b) & 0xFFFFFFFF) << (32 * l) for l, (a, b) in enumerate(zip(_lanes(v), _lanes(cw))))
    return _lanes(seed)


def eval_full_flat_et(orc, key, prf):
    """share of every row, natural order, int32 [n]"""
    d = key_depth(key)
    out = np.zeros(4 << d, np.uint32)
    for j in range(1 << d):
        out[4 * j:4 * j + 4] = eval_flat_et(orc, key, j, prf)
    return out.view(np.int32)


def eval_dot_et(orc, keys, prf, table):
    """out[b][e] = sum_i share_b[i] * table[i][e] mod 2^32, int32 [B, E]"""
    keys = np.asarray(keys, np.int32).reshape(-1, KEY_WORDS)
    return dot_u32(np.stack([eval_full_flat_et(orc, k, prf) for k in keys]), table)


def dot_u32(shares, table):
    """int32 share vectors [B, n] x int32 table [n, E] -> int32 [B, E], wrapping mod 2^32"""
    s = np.asarray(shares, np.int32).view(np.uint32).astype(np.uint64)
    t = np.asarray(table, np.int32).view(np.uint32).astype(np.uint64)
    out = np.zeros((s.shape[0], t.shape[1]), np.uint64)
    for e in range(t.shape[1]):
        out[:, e] = ((s * t[:, e][None, :]) & np.uint64(0xFFFFFFFF)).sum(axis=1) & np.uint64(0xFFFFFFFF)
    return out.astype(np.uint32).view(np.int32)
