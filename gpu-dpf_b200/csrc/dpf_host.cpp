/*
 * dpf_host.cpp -- CPU side of the API: key generation (client) and eval_cpu.
 *
 * Mirrors the CPU entry points of the reference extension:
 *   gen       dpf_wrapper.cu:49-68  -> dpf_base/dpf.h:403-464 (log construction),
 *                                      :290-360 (N=2 base), :239-270 (flatten)
 *   eval_cpu  dpf_wrapper.cu:70-84  -> dpf_base/dpf.h:362-377 (EvaluateFlat)
 * Written against the definitions, using the shared arithmetic core
 * (dpf_core.cuh) for the PRFs.
 */
#include "dpf_host.h"

#include <cstring>
#include <mutex>
#include <random>
#include <utility>
#include <vector>

namespace b200dpf {
namespace host {

typedef unsigned __int128 u128;

namespace {

uint8_t g_sbox[256];
uint32_t g_te0[256];
std::once_flag g_tables_once;

uint8_t rotl8(uint8_t v, int r) { return (uint8_t)((v << r) | (v >> (8 - r))); }

void build_tables()
{
    /* S-box by walking the multiplicative group of GF(2^8) with generator 3
     * (p) and its inverse (q), then the FIPS-197 affine map. */
    uint8_t p = 1, q = 1;
    do {
        p = (uint8_t)(p ^ (p << 1) ^ ((p & 0x80) ? 0x1b : 0));
        q ^= (uint8_t)(q << 1);
        q ^= (uint8_t)(q << 2);
        q ^= (uint8_t)(q << 4);
        if (q & 0x80) q ^= 0x09;
        g_sbox[p] = (uint8_t)(q ^ rotl8(q, 1) ^ rotl8(q, 2) ^ rotl8(q, 3) ^ rotl8(q, 4) ^ 0x63);
    } while (p != 1);
    g_sbox[0] = 0x63;
    for (int v = 0; v < 256; v++) {
        const uint32_t s = g_sbox[v];
        const uint32_t s2 = ((s << 1) ^ ((s & 0x80) ? 0x11b : 0)) & 0xff;
        const uint32_t s3 = s2 ^ s;
        g_te0[v] = s2 | (s << 8) | (s << 16) | (s3 << 24);
    }
}

u128 to_u128(const Seed &s)
{
    return ((u128)s.w << 96) | ((u128)s.z << 64) | ((u128)s.y << 32) | (u128)s.x;
}

Seed from_u128(u128 v)
{
    return make_seed((uint32_t)v, (uint32_t)(v >> 32), (uint32_t)(v >> 64), (uint32_t)(v >> 96));
}

void set_slot(int32_t *key, int slot, u128 v)
{
    std::memcpy(reinterpret_cast<uint8_t *>(key) + 16 * (size_t)slot, &v, 16);
}

u128 prf128(int prf_id, u128 seed, uint32_t pos) { return to_u128(prf(prf_id, from_u128(seed), pos)); }

/* The reference's generator: std::mt19937 behind the draws of dpf_base/dpf.h:272-283
 * (128-bit = two 64-bit uniform draws, high half first) and :450 (32-bit upper-level words). */
struct ReferenceRng {
    std::mt19937 g;
    explicit ReferenceRng(uint32_t seed32) : g(seed32) {}
    u128 draw128()
    {
        std::uniform_int_distribution<uint64_t> d(0, std::numeric_limits<uint64_t>::max());
        const uint64_t hi = d(g);
        const uint64_t lo = d(g);
        return ((u128)hi << 64) | lo;
    }
    u128 draw_upper_cw() { return (u128)g(); }
};

/* ChaCha20 (RFC 8439 block function) keystream as a deterministic random bit generator. */
struct ChaCha20Rng {
    uint32_t state[16];
    uint32_t block[16];
    int used = 16;
    ChaCha20Rng(const uint8_t key[32], const uint8_t nonce[12])
    {
        static const uint32_t sigma[4] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u};
        for (int i = 0; i < 4; i++) state[i] = sigma[i];
        for (int i = 0; i < 8; i++) std::memcpy(&state[4 + i], key + 4 * i, 4);
        state[12] = 0;
        for (int i = 0; i < 3; i++) std::memcpy(&state[13 + i], nonce + 4 * i, 4);
    }
    static uint32_t rl(uint32_t v, int r) { return (v << r) | (v >> (32 - r)); }
    static void qr(uint32_t *x, int a, int b, int c, int d)
    {
        x[a] += x[b]; x[d] = rl(x[d] ^ x[a], 16);
        x[c] += x[d]; x[b] = rl(x[b] ^ x[c], 12);
        x[a] += x[b]; x[d] = rl(x[d] ^ x[a], 8);
        x[c] += x[d]; x[b] = rl(x[b] ^ x[c], 7);
    }
    void refill()
    {
        uint32_t x[16];
        std::memcpy(x, state, sizeof x);
        for (int r = 0; r < 10; r++) {
            qr(x, 0, 4, 8, 12); qr(x, 1, 5, 9, 13); qr(x, 2, 6, 10, 14); qr(x, 3, 7, 11, 15);
            qr(x, 0, 5, 10, 15); qr(x, 1, 6, 11, 12); qr(x, 2, 7, 8, 13); qr(x, 3, 4, 9, 14);
        }
        for (int i = 0; i < 16; i++) block[i] = x[i] + state[i];
        state[12]++;
        used = 0;
    }
    uint32_t draw32()
    {
        if (used == 16) refill();
        return block[used++];
    }
    u128 draw128()
    {
        u128 v = 0;
        for (int i = 0; i < 4; i++) v |= (u128)draw32() << (32 * i);
        return v;
    }
    u128 draw_upper_cw() { return draw128(); }
};

template <class Rng>
u128 random128_odd(Rng &g)
{
    u128 k = 0;
    while ((k & 1) == 0) k = g.draw128();
    return k;
}

/* GROUP (dpf_core.cuh) is the group of flat level 0, where the payload lives: Z/2^128 for standard
 * keys, lane-wise (Z/2^32)^4 for early-terminated keys, (Z/2)^128 for XOR-shared keys, whose add and
 * subtract are both XOR (level0_add / level0_sub).  Every other level adds in Z/2^128. */
template <class Rng, int GROUP = GROUP_ADD128>
struct KeyBuilder {
    int depth;
    int64_t alpha;
    int prf_id;
    Rng &g;
    u128 cw1[64], cw2[64];
    u128 root_a, root_b;

    u128 add(int L, u128 a, u128 b) const { return L == 0 ? level0_add<GROUP>(a, b) : a + b; }
    u128 sub(int L, u128 a, u128 b) const { return L == 0 ? level0_sub<GROUP>(a, b) : a - b; }

    /* Builds flat level L (domain 2^(depth-L)) for payload `beta` and returns
     * the two servers' seeds on the alpha path just below this level. */
    std::pair<u128, u128> build(int L, u128 beta)
    {
        const int row = (int)((alpha >> (depth - 1 - L)) & 1);
        u128 up_a, up_b;   /* seeds entering this level on the alpha path */
        if (L == depth - 1) {
            /* N = 2 base: one seed per server, differing in the LSB (dpf.h:318-331) */
            u128 ka = g.draw128(), kb = g.draw128();
            ka &= ~(u128)1;
            kb = (kb & ~(u128)1) | 1;
            root_a = ka;
            root_b = kb;
            u128 delta[2];
            for (int i = 0; i < 2; i++) {
                delta[i] = sub(L, prf128(prf_id, ka, (uint32_t)i), prf128(prf_id, kb, (uint32_t)i));
                if (i == row) delta[i] = sub(L, delta[i], beta);
            }
            for (int i = 0; i < 2; i++) {
                cw1[2 * L + i] = g.draw128();
                cw2[2 * L + i] = add(L, cw1[2 * L + i], delta[i]);
            }
            up_a = ka;
            up_b = kb;
        } else {
            const u128 beta_below = random128_odd(g);
            const std::pair<u128, u128> below = build(L + 1, beta_below);
            up_a = below.first;
            up_b = below.second;
            const bool a_even = (up_a & 1) == 0;
            for (int i = 0; i < 2; i++) {
                u128 d = sub(L, prf128(prf_id, up_b, (uint32_t)i), prf128(prf_id, up_a, (uint32_t)i));
                if (a_even) d = sub(L, 0, d);
                cw1[2 * L + i] = g.draw_upper_cw();   /* reference: a 32-bit draw, dpf.h:450 */
                cw2[2 * L + i] = add(L, cw1[2 * L + i], d);
                if (i == row) cw1[2 * L + i] = a_even ? add(L, cw1[2 * L + i], beta) : sub(L, cw1[2 * L + i], beta);
            }
        }
        const u128 *bank_a = (up_a & 1) ? cw2 : cw1;
        const u128 *bank_b = (up_b & 1) ? cw2 : cw1;
        return std::make_pair(prf128(prf_id, up_a, (uint32_t)row) + bank_a[2 * L + row],
                              prf128(prf_id, up_b, (uint32_t)row) + bank_b[2 * L + row]);
    }
};

}  // namespace

const uint32_t *aes_te0()
{
    std::call_once(g_tables_once, build_tables);
    return g_te0;
}

const uint8_t *aes_sbox()
{
    std::call_once(g_tables_once, build_tables);
    return g_sbox;
}

Seed prf(int prf_id, const Seed &s, uint32_t pos)
{
    AesHostTables ta;
    ta.te0 = (prf_id == PRF_AES128) ? aes_te0() : nullptr;
    switch (prf_id) {
    case PRF_DUMMY: return expand_one<PRF_DUMMY>(ta, s, pos);
    case PRF_SALSA20: return expand_one<PRF_SALSA20>(ta, s, pos);
    case PRF_CHACHA20: return expand_one<PRF_CHACHA20>(ta, s, pos);
    default: return expand_one<PRF_AES128>(ta, s, pos);
    }
}

int key_depth(const int32_t *key, int kind)
{
    const KindInfo &k = kKinds[kind];
    const Seed d = key_slot(key, SLOT_DEPTH);
    if (d.y != (uint32_t)k.lane_bits || d.z || d.w || d.x < 1 || d.x > (uint32_t)k.max_depth) return -1;
    return (int)d.x;
}

/* slot 130 = 2^(depth + lane_bits) as a u64: a standard key of depth 32 has n = 2^32, and the other kinds
 * (n <= 2^31) a zero high word */
int64_t key_n(const int32_t *key, int kind)
{
    const Seed v = key_slot(key, SLOT_N);
    const int depth = key_depth(key, kind);
    if (depth < 0 || v.z || v.w) return -1;
    const int64_t n = ((int64_t)v.y << 32) | v.x;
    if (n != ((int64_t)1 << (depth + kKinds[kind].lane_bits))) return -1;
    return n;
}

int key_kind(const int32_t *key)
{
    const uint32_t lane_bits = key_slot(key, SLOT_DEPTH).y;
    for (int kind = 0; kind < KIND_COUNT; kind++)
        if (lane_bits == (uint32_t)kKinds[kind].lane_bits) return key_n(key, kind) >= 0 ? kind : -1;
    return -1;
}

namespace {

template <class Rng>
int gen_with(Rng &rng, int64_t alpha, int64_t n, int prf_id, int32_t *key_a, int32_t *key_b)
{
    if (n < 2 || (n & (n - 1)) != 0 || alpha < 0 || alpha >= n) return -1;
    if (prf_id < PRF_DUMMY || prf_id > PRF_AES128) return -1;
    int depth = 0;
    while (((int64_t)1 << depth) < n) depth++;
    if (depth > 32) return -1;

    KeyBuilder<Rng> kb{depth, alpha, prf_id, rng, {}, {}, 0, 0};
    std::memset(kb.cw1, 0, sizeof kb.cw1);
    std::memset(kb.cw2, 0, sizeof kb.cw2);
    kb.build(0, (u128)1);   /* beta = 1, dpf_wrapper.cu:53 */

    for (int srv = 0; srv < 2; srv++) {
        int32_t *key = srv ? key_b : key_a;
        std::memset(key, 0, sizeof(int32_t) * KEY_WORDS);
        set_slot(key, SLOT_DEPTH, (u128)depth);
        for (int i = 0; i < 64; i++) {
            set_slot(key, SLOT_CW1 + i, kb.cw1[i]);
            set_slot(key, SLOT_CW2 + i, kb.cw2[i]);
        }
        set_slot(key, SLOT_ROOT, srv ? kb.root_b : kb.root_a);
        set_slot(key, SLOT_N, (u128)n);
    }
    return 0;
}

}  // namespace

int gen(int64_t alpha, int64_t n, uint32_t seed32, int prf_id, int32_t *key_a, int32_t *key_b)
{
    ReferenceRng rng(seed32);   /* dpf_wrapper.cu:52: only 32 bits of the seed reach the engine */
    return gen_with(rng, alpha, n, prf_id, key_a, key_b);
}

int gen_secure(int64_t alpha, int64_t n, const uint8_t seed[44], int prf_id, int32_t *key_a, int32_t *key_b)
{
    ChaCha20Rng rng(seed, seed + 32);
    return gen_with(rng, alpha, n, prf_id, key_a, key_b);
}

namespace {

/* A key whose leaves carry 2^lane_bits table rows each (early-terminated: 4, XOR-shared: 128): the log
 * construction over the 2^depth leaves for alpha >> lane_bits, level 0 in GROUP, payload beta. */
template <int GROUP>
int gen_leaves_in(const KindInfo &k, int64_t alpha, int64_t n, const uint8_t seed[44], int prf_id, int32_t *key_a,
                  int32_t *key_b, u128 beta)
{
    if (n < k.n_min || n > k.n_max || (n & (n - 1)) != 0 || alpha < 0 || alpha >= n) return -1;
    if (prf_id < PRF_DUMMY || prf_id > PRF_AES128) return -1;
    int depth = 0;
    while (((int64_t)1 << (depth + k.lane_bits)) < n) depth++;

    ChaCha20Rng rng(seed, seed + 32);
    KeyBuilder<ChaCha20Rng, GROUP> kb{depth, alpha >> k.lane_bits, prf_id, rng, {}, {}, 0, 0};
    std::memset(kb.cw1, 0, sizeof kb.cw1);
    std::memset(kb.cw2, 0, sizeof kb.cw2);
    kb.build(0, beta);

    for (int srv = 0; srv < 2; srv++) {
        int32_t *key = srv ? key_b : key_a;
        std::memset(key, 0, sizeof(int32_t) * KEY_WORDS);
        set_slot(key, SLOT_DEPTH, (u128)depth | ((u128)k.lane_bits << 32));
        for (int i = 0; i < 64; i++) {
            set_slot(key, SLOT_CW1 + i, kb.cw1[i]);
            set_slot(key, SLOT_CW2 + i, kb.cw2[i]);
        }
        set_slot(key, SLOT_ROOT, srv ? kb.root_b : kb.root_a);
        set_slot(key, SLOT_N, (u128)n);
    }
    return 0;
}

}  // namespace

int gen_leaves(int kind, int64_t alpha, int64_t n, const uint8_t seed[44], int prf_id, int32_t *key_a, int32_t *key_b)
{
    const KindInfo &k = kKinds[kind];
    /* beta = unit vector of 32-bit lane alpha & 3, or of bit alpha & 127 */
    if (kind == KIND_ET)
        return gen_leaves_in<kKinds[KIND_ET].group>(k, alpha, n, seed, prf_id, key_a, key_b, (u128)1 << (32 * (alpha & 3)));
    if (kind == KIND_XOR)
        return gen_leaves_in<kKinds[KIND_XOR].group>(k, alpha, n, seed, prf_id, key_a, key_b, (u128)1 << (alpha & 127));
    return -1;
}

namespace {

/* per-key storage for the CPU traversal */
struct CpuEnv {
    AesHostTables ta;
    const int32_t *key;
    int depth;
    Seed stack[33];
    uint32_t base_pos;
    int32_t *out;

    Seed cw(int level, uint32_t bank, uint32_t bit) const
    {
        return key_slot(key, (bank ? SLOT_CW2 : SLOT_CW1) + 2 * level + (int)bit);
    }
    uint32_t cw_lo(uint32_t bank, uint32_t bit) const { return cw(0, bank, bit).x; }
    void push(int h, const Seed &s) { stack[h] = s; }
    Seed pop(int h) const { return stack[h]; }
    void leaf_prefetch(uint32_t) {}
    void node_pair(uint32_t, const Seed &, const Seed &) {}
    void leaf_pair(uint32_t local_pos, uint32_t v0, uint32_t v1)
    {
        /* position p holds index bitrev_depth(p) */
        out[bitrev(base_pos + local_pos, depth)] = (int32_t)v0;
        out[bitrev(base_pos + local_pos + 1, depth)] = (int32_t)v1;
    }
    void leaf_quads(uint32_t local_pos, const Seed &w0, const Seed &w1)
    {
        /* leaf position p holds leaf bitrev_depth(p), whose word l is out[4 * leaf + l]: the share of row
         * 4 * leaf + l (early-terminated), or the packed share bits of rows 128 * leaf + 32 l .. +31 (XOR) */
        int32_t *o0 = out + 4 * (size_t)bitrev(base_pos + local_pos, depth);
        int32_t *o1 = out + 4 * (size_t)bitrev(base_pos + local_pos + 1, depth);
        o0[0] = (int32_t)w0.x; o0[1] = (int32_t)w0.y; o0[2] = (int32_t)w0.z; o0[3] = (int32_t)w0.w;
        o1[0] = (int32_t)w1.x; o1[1] = (int32_t)w1.y; o1[2] = (int32_t)w1.z; o1[3] = (int32_t)w1.w;
    }
};

template <int PRF>
void eval_cpu_impl(const int32_t *key, int group, int depth, int32_t *out)
{
    CpuEnv env;
    env.ta.te0 = aes_te0();
    env.key = key;
    env.depth = depth;
    env.out = out;
    /* 2^s-leaf subtrees, s <= 16, walked to from the root one after another */
    const int s = depth < 16 ? depth : 16;
    const uint32_t nsub = 1u << (depth - s);
    for (uint32_t q = 0; q < nsub; q++) {
        env.base_pos = q << s;
        const Seed r = walk_down<PRF>(env, key_slot(key, SLOT_ROOT), depth - 1, depth - s, q);
        if (group == GROUP_XOR128) eval_subtree<PRF, false, CpuEnv, GROUP_XOR128>(env, r, s, 0);
        else if (group == GROUP_LANES32) eval_subtree<PRF, false, CpuEnv, GROUP_LANES32>(env, r, s, 0);
        else eval_subtree<PRF, false, CpuEnv, GROUP_ADD128>(env, r, s, 0);
    }
}

}  // namespace

int eval_cpu(const int32_t *key, int kind, int prf_id, int32_t *out)
{
    const int depth = key_depth(key, kind);
    /* a standard key of depth 32 has 2^32 rows, more than the output can hold */
    if (depth < 1 || (kind == KIND_STANDARD && depth > 31) || key_n(key, kind) < 0) return -1;
    const int group = kKinds[kind].group;
    switch (prf_id) {
    case PRF_DUMMY: eval_cpu_impl<PRF_DUMMY>(key, group, depth, out); break;
    case PRF_SALSA20: eval_cpu_impl<PRF_SALSA20>(key, group, depth, out); break;
    case PRF_CHACHA20: eval_cpu_impl<PRF_CHACHA20>(key, group, depth, out); break;
    case PRF_AES128: eval_cpu_impl<PRF_AES128>(key, group, depth, out); break;
    default: return -2;
    }
    return 0;
}

}  // namespace host
}  // namespace b200dpf
