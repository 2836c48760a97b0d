"""Key generation restated in plain Python, for the tests: every key kind, both random sources.

Written from the documented construction (include/b200dpf.h: b200dpf_gen_secure, _gen_et, _gen_xor and the
compact form; DESIGN.md sections 8, 9 and 10), not from the engine's generators.  It is trusted because of its
anchors in tests/test_keygen_ref_host.py: the ChaCha20 block function reproduces RFC 8439's test vectors, and the
construction, driven by the reference's mt19937 stream, reproduces the reference's own keys.

Draw sources (one per key pair):
  ChaCha20Drbg(seed)   the RFC 8439 block function keyed with seed[0:32], nonce seed[32:44], block counter from 0;
                       a block is 16 little-endian words, a 128-bit draw is 4 words, low word first.
  MT19937Draws(seed32) std::mt19937 seeded with seed32, as the reference draws from it: a 128-bit draw is two
                       64-bit halves, high half first, each half two outputs with the first one high; an
                       upper-level correction word is one 32-bit output.
Both draw an odd 128-bit value by rejecting even draws and drawing again.

The construction (the reference's log(n) recursion over its N = 2 base case), for a tree of depth d over the
2^d leaves and the leaf alpha >> lane_bits:
  1. payloads: an odd draw for each level 1 .. d-1, top-down (level 0's payload is beta);
  2. the N = 2 base at level d-1: root seeds k_a = draw with LSB 0, k_b = draw with LSB 1;
     delta[i] = PRF(k_a, i) - PRF(k_b, i), minus the level's payload at i = the leaf's bit 0;
     cw_1[i] = draw, cw_2[i] = cw_1[i] + delta[i];
  3. on the way up, levels d-2 .. 0, from the two servers' seeds s_a, s_b on the alpha path below the level:
     diff[i] = PRF(s_b, i) - PRF(s_a, i), negated when s_a is even; cw_1[i] = draw, cw_2[i] = cw_1[i] + diff[i];
     at i = the leaf's bit (d-1-L), cw_1[i] += payload if s_a is even, else -= payload.
  A server's seed below level L is PRF(s, bit) + (cw_2 if s is odd else cw_1)[bit].
Level 0 adds in the kind's group (Z/2^128, (Z/2^32)^4 lane-wise, or (Z/2)^128 as XOR); every other level in
Z/2^128.  beta is 1, 1 << 32 * (alpha & 3) or 1 << (alpha & 127).
"""
import collections
import hashlib
import struct

import numpy as np

M32 = (1 << 32) - 1
M128 = (1 << 128) - 1
KEY_WORDS = 524


# ---- ChaCha20 (RFC 8439 section 2.3) -------------------------------------------------------------------------

def _rotl(v, r):
    return ((v << r) | (v >> (32 - r))) & M32


def _quarter(x, a, b, c, d):
    x[a] = (x[a] + x[b]) & M32
    x[d] = _rotl(x[d] ^ x[a], 16)
    x[c] = (x[c] + x[d]) & M32
    x[b] = _rotl(x[b] ^ x[c], 12)
    x[a] = (x[a] + x[b]) & M32
    x[d] = _rotl(x[d] ^ x[a], 8)
    x[c] = (x[c] + x[d]) & M32
    x[b] = _rotl(x[b] ^ x[c], 7)


def chacha20_block(key, counter, nonce):
    """RFC 8439 section 2.3.2: the 16 output words of the block function for a 32-byte key, a 32-bit block
    counter and a 12-byte nonce"""
    state = [0x61707865, 0x3320646E, 0x79622D32, 0x6B206574]
    state += list(struct.unpack("<8I", bytes(key)))
    state += [counter & M32]
    state += list(struct.unpack("<3I", bytes(nonce)))
    x = list(state)
    for _ in range(10):
        _quarter(x, 0, 4, 8, 12)
        _quarter(x, 1, 5, 9, 13)
        _quarter(x, 2, 6, 10, 14)
        _quarter(x, 3, 7, 11, 15)
        _quarter(x, 0, 5, 10, 15)
        _quarter(x, 1, 6, 11, 12)
        _quarter(x, 2, 7, 8, 13)
        _quarter(x, 3, 4, 9, 14)
    return [(x[i] + state[i]) & M32 for i in range(16)]


def chacha20_block_bytes(key, counter, nonce):
    """the serialised block: its words little endian"""
    return struct.pack("<16I", *chacha20_block(key, counter, nonce))


# ---- draw sources --------------------------------------------------------------------------------------------

class _Draws:
    """What every draw source counts: blocks (or outputs) consumed and the rejections of each odd draw"""

    def __init__(self):
        self.odd_rejections = []     # per odd draw, in order: how many even values it rejected

    def draw_odd(self):
        rejected = 0
        v = self.draw128()
        while v & 1 == 0:
            rejected += 1
            v = self.draw128()
        self.odd_rejections.append(rejected)
        return v

    @property
    def rejections(self):
        return sum(self.odd_rejections)


class ChaCha20Drbg(_Draws):
    """the ChaCha20 keystream of the first 44 seed bytes (key || nonce) as a source of 128-bit draws"""

    def __init__(self, seed):
        super().__init__()
        seed = bytes(seed)
        if len(seed) < 44:
            raise ValueError("a ChaCha20 DRBG takes at least 44 seed bytes")
        self.key, self.nonce = seed[:32], seed[32:44]
        self.blocks = 0              # keystream blocks generated so far; the next one has this counter
        self._words = []

    def _word(self):
        if not self._words:
            self._words = chacha20_block(self.key, self.blocks, self.nonce)
            self.blocks += 1
        return self._words.pop(0)

    def draw128(self):
        v = 0
        for i in range(4):
            v |= self._word() << (32 * i)
        return v

    draw_upper_cw = draw128


class MT19937Draws(_Draws):
    """the reference's generator: std::mt19937 seeded with a 32-bit value.  numpy's legacy RandomState seeds the
    same generator the same way, and random_raw() returns its 32-bit outputs in order."""

    def __init__(self, seed32):
        super().__init__()
        self._bg = np.random.RandomState(seed32 & M32)._bit_generator
        self.outputs = 0

    def output(self):
        self.outputs += 1
        return int(self._bg.random_raw())

    def _draw64(self):
        hi = self.output()
        return (hi << 32) | self.output()

    def draw128(self):
        hi = self._draw64()
        return (hi << 64) | self._draw64()

    def draw_upper_cw(self):
        return self.output()


# ---- level-0 groups and kinds --------------------------------------------------------------------------------

def _lanes(v):
    return [(v >> (32 * i)) & M32 for i in range(4)]


def _from_lanes(w):
    return sum((x & M32) << (32 * i) for i, x in enumerate(w))


ADD128, LANES32, XOR128 = "Z/2^128", "(Z/2^32)^4", "(Z/2)^128"


def group_add(group, a, b):
    if group == ADD128:
        return (a + b) & M128
    if group == LANES32:
        return _from_lanes([x + y for x, y in zip(_lanes(a), _lanes(b))])
    return a ^ b


def group_sub(group, a, b):
    if group == ADD128:
        return (a - b) & M128
    if group == LANES32:
        return _from_lanes([x - y for x, y in zip(_lanes(a), _lanes(b))])
    return a ^ b


Kind = collections.namedtuple("Kind", "name lane_bits group magic n_min n_max")
KINDS = {
    "standard": Kind("standard", 0, ADD128, b"DPF2", 2, 1 << 32),
    "et": Kind("early-terminated", 2, LANES32, b"DPE4", 8, 1 << 31),
    "xor": Kind("XOR-shared", 7, XOR128, b"DPX7", 256, 1 << 31),
}


def beta0(kind, alpha):
    """the payload at level 0: the value the two servers' leaf outputs at alpha differ by"""
    if kind == "et":
        return 1 << (32 * (alpha & 3))
    if kind == "xor":
        return 1 << (alpha & 127)
    return 1


def depth_of(kind, n):
    return n.bit_length() - 1 - KINDS[kind].lane_bits


def max_depth(kind):
    return depth_of(kind, KINDS[kind].n_max)


# ---- the construction ----------------------------------------------------------------------------------------

_ORACLE = None


def oracle_prf(prf, seed, pos):
    """the PRFs of oracle/dpf_oracle.c, which tests/test_oracle.py pins to the reference's"""
    global _ORACLE
    if _ORACLE is None:
        import oracle
        _ORACLE = oracle.Oracle()
    return _ORACLE.prf(prf, seed, pos)


Keys = collections.namedtuple("Keys", "a b packed_a packed_b draws")


def build(depth, leaf, beta, group, prf, draws, prf_fn=oracle_prf):
    """(root_a, root_b, cw1, cw2): the two root seeds and the correction words cw1[2L + i], cw2[2L + i] of flat
    levels L = 0 .. depth-1 of a tree over 2^depth leaves with the point at `leaf`"""
    F = lambda s, i: prf_fn(prf, s, i)  # noqa: E731
    add = lambda L, a, b: group_add(group, a, b) if L == 0 else (a + b) & M128  # noqa: E731
    sub = lambda L, a, b: group_sub(group, a, b) if L == 0 else (a - b) & M128  # noqa: E731
    bit = lambda L: (leaf >> (depth - 1 - L)) & 1  # noqa: E731
    payload = [beta] + [draws.draw_odd() for _ in range(1, depth)]
    cw1, cw2 = [0] * (2 * depth), [0] * (2 * depth)

    def below(L, s):
        """a server's seed below level L on the alpha path"""
        b = bit(L)
        return (F(s, b) + (cw2 if s & 1 else cw1)[2 * L + b]) & M128

    L = depth - 1
    root_a = draws.draw128() & ~1
    root_b = draws.draw128() | 1
    delta = [sub(L, F(root_a, i), F(root_b, i)) for i in range(2)]
    delta[bit(L)] = sub(L, delta[bit(L)], payload[L])
    for i in range(2):
        cw1[2 * L + i] = draws.draw128()
        cw2[2 * L + i] = add(L, cw1[2 * L + i], delta[i])
    s_a, s_b = root_a, root_b
    for L in range(depth - 2, -1, -1):
        s_a, s_b = below(L + 1, s_a), below(L + 1, s_b)
        even = s_a & 1 == 0
        for i in range(2):
            diff = sub(L, F(s_b, i), F(s_a, i))
            if even:
                diff = sub(L, 0, diff)
            cw1[2 * L + i] = draws.draw_upper_cw()
            cw2[2 * L + i] = add(L, cw1[2 * L + i], diff)
            if i == bit(L):
                cw1[2 * L + i] = (add if even else sub)(L, cw1[2 * L + i], payload[L])
    return root_a, root_b, cw1, cw2


def _slot(v):
    return np.frombuffer(int(v).to_bytes(16, "little"), np.int32)


def wire_key(kind, depth, root, cw1, cw2):
    """int32[524]: 131 little-endian 128-bit slots, [0] = (depth, lane_bits, 0, 0), [1 + j] = cw_1[j],
    [65 + j] = cw_2[j], [129] = root seed, [130] = n; every other slot zero"""
    k = KINDS[kind]
    key = np.zeros((131, 4), np.int32)
    key[0] = _slot(depth | (k.lane_bits << 32))
    for j in range(2 * depth):
        key[1 + j] = _slot(cw1[j])
        key[65 + j] = _slot(cw2[j])
    key[129] = _slot(root)
    key[130] = _slot(1 << (depth + k.lane_bits))
    return key.reshape(KEY_WORDS)


def compact_key(kind, depth, root, cw1, cw2):
    """the kind's compact form: magic | depth (u8) | 11 zero bytes | root | per level L: cw_1[2L], cw_1[2L+1],
    cw_2[2L], cw_2[2L+1] (16 bytes each, little endian) -- 32 + 64 * depth bytes"""
    out = KINDS[kind].magic + bytes([depth]) + bytes(11) + root.to_bytes(16, "little")
    for L in range(depth):
        for v in (cw1[2 * L], cw1[2 * L + 1], cw2[2 * L], cw2[2 * L + 1]):
            out += v.to_bytes(16, "little")
    return out


def gen_with(kind, alpha, n, prf, draws, prf_fn=oracle_prf):
    """both servers' keys of `kind` for row alpha of an n-row table, every random value from `draws`"""
    k = KINDS[kind]
    if not (k.n_min <= n <= k.n_max and n & (n - 1) == 0 and 0 <= alpha < n):
        raise ValueError("no %s key for alpha=%d, n=%d" % (k.name, alpha, n))
    depth = depth_of(kind, n)
    root_a, root_b, cw1, cw2 = build(depth, alpha >> k.lane_bits, beta0(kind, alpha), k.group, prf, draws, prf_fn)
    return Keys(wire_key(kind, depth, root_a, cw1, cw2), wire_key(kind, depth, root_b, cw1, cw2),
                compact_key(kind, depth, root_a, cw1, cw2), compact_key(kind, depth, root_b, cw1, cw2), draws)


def gen(kind, alpha, n, seed, prf, prf_fn=oracle_prf):
    """the ChaCha20-DRBG keys of `kind` (b200dpf_gen_secure, _gen_et, _gen_xor) from the first 44 seed bytes"""
    return gen_with(kind, alpha, n, prf, ChaCha20Drbg(seed), prf_fn)


def gen_mt(alpha, n, seed32, prf, prf_fn=oracle_prf):
    """the reference generator's standard keys (b200dpf_gen)"""
    return gen_with("standard", alpha, n, prf, MT19937Draws(seed32), prf_fn)


# ---- rows and seeds at the edges -----------------------------------------------------------------------------

# rows at the edges of a leaf: its first and last, and for XOR-shared keys the edges of its 32-bit words
LANE_EDGES = {"standard": (), "et": (0, 3), "xor": (0, 31, 32, 127)}


def edge_rows(kind, n, rng):
    """0, n - 1, the lane edges of one random leaf and one random row (rng: a random.Random)"""
    lane_bits = KINDS[kind].lane_bits
    leaf = rng.randrange(n >> lane_bits)
    rows = [0, n - 1] + [(leaf << lane_bits) | e for e in LANE_EDGES[kind]] + [rng.randrange(n)]
    return list(dict.fromkeys(rows))


def payload_rejections(seed, depth):
    """the rejections of each payload draw of a depth-`depth` key from `seed`: the payloads are the key's first
    draws, so they do not depend on alpha, n, the kind or the PRF"""
    g = ChaCha20Drbg(seed)
    for _ in range(depth - 1):
        g.draw_odd()
    return g.odd_rejections


def search_seed(depth, accept, tag):
    """the first seed of a fixed sequence whose payload rejections at `depth` satisfy `accept`"""
    for i in range(1 << 16):
        seed = hashlib.sha512(b"%s %d %d" % (tag.encode(), depth, i)).digest()[:44]
        if accept(payload_rejections(seed, depth)):
            return seed
    raise AssertionError("no seed found for %s at depth %d" % (tag, depth))


Coverage = collections.namedtuple("Coverage", "name depth seed")


def coverage_seeds(kind):
    """seeds whose keys take the DRBG through its edges, for keys of `kind`:
      depth 1        no payloads at all: the key is the N = 2 base alone;
      depth 2        the only payload (also the last) rejects two even draws in a row;
      deepest        the last payload rejects at least once, an earlier one at least twice, and the key runs
                     past 16 keystream blocks."""
    d = max_depth(kind)
    return [
        Coverage("depth 1", 1, search_seed(1, lambda r: r == [], "depth 1")),
        Coverage("two rejections", 2, search_seed(2, lambda r: r[-1] >= 2, "two rejections")),
        Coverage("deepest", d, search_seed(d, lambda r: r[-1] >= 1 and max(r[:-1]) >= 2, "deepest")),
    ]
