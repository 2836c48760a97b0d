"""Per-index oracle for XOR-shared DPF keys -- TEST INFRASTRUCTURE ONLY.

These functions restate the definition of XOR-shared keys (DESIGN.md section 10) and share no code
with the engine's tree walk: every leaf is reached by its own root-to-leaf walk, one PRF call per
level, through the pinned PRF of the C oracle (oracle/dpf_oracle.c, ``orc_prf``).  The reference has
no such keys; what pins the construction is that the two servers' share bits XOR to the one-hot
vector of alpha, and the golden file tests/golden/xor_v1.npz.

    leaf j = i >> 7, bit position b = i & 127, tree depth d = log2(n) - 7
    step k = 0 .. d-1 consumes bit k of j (the root takes the least significant bit) with
    correction-word level L = d-1-k, bank cw_2 when the parent seed is odd, else cw_1:
        child = PRF(parent, bit) + cw[2L + bit]   mod 2^128, for L > 0
        child = PRF(parent, bit) XOR cw[2L + bit]            for L = 0  (the group (Z/2)^128)
    share[i] = bit b of the leaf value (bit b of a 128-bit value: bit b & 31 of little-endian word b >> 5)
    result[e] = XOR over i of (share[i] ? table[i][e] : 0)
"""
import numpy as np

KEY_WORDS = 524
M128 = (1 << 128) - 1


def _slot(key, s):
    w = np.asarray(key, np.int32).view(np.uint32)[4 * s:4 * s + 4]
    return int(w[0]) | int(w[1]) << 32 | int(w[2]) << 64 | int(w[3]) << 96


def key_depth(key):
    """tree depth d of an XOR-shared key (slot 0 = (d, 7, 0, 0)), n = 128 * 2^d rows"""
    k = np.asarray(key, np.int32)
    assert int(k[1]) == 7 and int(k[2]) == 0 and int(k[3]) == 0, "not an XOR-shared key"
    d = int(k[0])
    assert _slot(k, 130) == 128 << d
    return d


def leaf_value(orc, key, leaf, prf):
    """the 128-bit value of leaf `leaf`, whose bit b is the share of row 128 * leaf + b"""
    d = key_depth(key)
    seed = _slot(key, 129)
    for k in range(d):
        bit = (leaf >> k) & 1
        level = d - 1 - k
        cw = _slot(key, (65 if seed & 1 else 1) + 2 * level + bit)
        v = orc.prf(prf, seed, bit)
        seed = (v + cw) & M128 if level > 0 else v ^ cw
    return seed


def share_bit(orc, key, i, prf):
    """the share bit of row i"""
    return (leaf_value(orc, key, i >> 7, prf) >> (i & 127)) & 1


def share_bits(orc, key, prf):
    """share bit of every row, natural order, uint8 [n]"""
    d = key_depth(key)
    out = np.zeros(128 << d, np.uint8)
    for j in range(1 << d):
        v = leaf_value(orc, key, j, prf)
        out[128 * j:128 * j + 128] = [(v >> b) & 1 for b in range(128)]
    return out


def pack_bits(bits):
    """share bits [n] -> uint32 [n / 32], row i = bit (i & 31) of word i >> 5 (eval_cpu_xor's layout)"""
    b = np.asarray(bits, np.uint8).reshape(-1, 32).astype(np.uint32)
    return (b << np.arange(32, dtype=np.uint32)).sum(axis=1, dtype=np.uint64).astype(np.uint32)


def unpack_bits(words):
    """uint32 [n / 32] -> share bits uint8 [n]"""
    w = np.asarray(words).view(np.uint32).reshape(-1, 1)
    return ((w >> np.arange(32, dtype=np.uint32)) & 1).astype(np.uint8).reshape(-1)


def xor_rows(bits, table):
    """XOR of the table rows whose bit is set: bits [B, n] (or [n]), int32 table [n, E] -> int32 [B, E]"""
    bits = np.atleast_2d(np.asarray(bits, np.uint8))
    t = np.asarray(table, np.int32).view(np.uint32)
    out = np.zeros((bits.shape[0], t.shape[1]), np.uint32)
    for b in range(bits.shape[0]):
        sel = t[bits[b].astype(bool)]
        if sel.shape[0]:
            out[b] = np.bitwise_xor.reduce(sel, axis=0)
    return out.view(np.int32)


def eval_xor(orc, keys, prf, table):
    """out[b][e] = XOR over i of (share_b[i] ? table[i][e] : 0), int32 [B, E]"""
    keys = np.asarray(keys, np.int32).reshape(-1, KEY_WORDS)
    return xor_rows(np.stack([share_bits(orc, k, prf) for k in keys]), table)
