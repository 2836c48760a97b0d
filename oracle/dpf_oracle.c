/*
 * oracle/dpf_oracle.c -- TEST INFRASTRUCTURE ONLY (see dpf_oracle.h).
 *
 * Plain-C restatement of the reference's CPU algorithm.  Written from the
 * algorithm's definition, not transcribed: the AES is a byte-oriented
 * FIPS-197 implementation with a computed S-box, key generation is an
 * iterative bottom-up loop instead of the reference's recursion, and the
 * Mersenne twister is restated from its published recurrence.  Equality with
 * the real reference is established by tests/test_oracle.py (PRFs, keygen incl. the
 * RNG stream, EvaluateFlat against oracle/_ref/libdpfref.so and tests/golden/golden_v1.npz).
 */
#include "dpf_oracle.h"

#include <pthread.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------ */
/* key wire format: dpf_wrapper.cu:26-46                                     */
/* ------------------------------------------------------------------------ */
enum { SLOT_DEPTH = 0, SLOT_CW1 = 1, SLOT_CW2 = 65, SLOT_ROOT = 129, SLOT_N = 130 };

static u128 key_slot(const int32_t *key, int slot)
{
    u128 v;
    memcpy(&v, (const uint8_t *)key + 16 * (size_t)slot, 16);
    return v;
}

static void key_set_slot(int32_t *key, int slot, u128 v)
{
    memcpy((uint8_t *)key + 16 * (size_t)slot, &v, 16);
}

static u128 mk128(uint64_t lo, uint64_t hi) { return ((u128)hi << 64) | lo; }

/* ------------------------------------------------------------------------ */
/* PRFs                                                                      */
/* ------------------------------------------------------------------------ */

/* dpf_base/dpf.h:72-74 */
static u128 prf_dummy(u128 seed, uint32_t pos)
{
    u128 k = (u128)pos + 4242;
    return seed * k + k;
}

static uint32_t rotl32(uint32_t v, int r) { return (v << r) | (v >> (32 - r)); }

/* The four "sigma" words as the reference spells them (dpf_base/dpf.h:102-105,
 * 163-166).  They are the byte-swapped form of the usual Salsa/ChaCha
 * constants, so no public test vector applies. */
static const uint32_t SIGMA[4] = { 0x65787061u, 0x6e642033u, 0x322d6279u, 0x7465206bu };

static void salsa_quarter(uint32_t *x, int a, int b, int c, int d)
{
    x[b] ^= rotl32(x[a] + x[d], 7);
    x[c] ^= rotl32(x[b] + x[a], 9);
    x[d] ^= rotl32(x[c] + x[b], 13);
    x[a] ^= rotl32(x[d] + x[c], 18);
}

/* dpf_base/dpf.h:84-135: Salsa20 core, 12 rounds, key words MSW first in
 * in[1..4], stream position in in[9]; PRF output = words 1..4 (word 1 = MSW). */
static u128 prf_salsa20_12(u128 seed, uint32_t pos)
{
    uint32_t in[16] = { 0 }, x[16];
    in[0] = SIGMA[0]; in[5] = SIGMA[1]; in[10] = SIGMA[2]; in[15] = SIGMA[3];
    in[1] = (uint32_t)(seed >> 96);
    in[2] = (uint32_t)(seed >> 64);
    in[3] = (uint32_t)(seed >> 32);
    in[4] = (uint32_t)seed;
    in[9] = pos;
    memcpy(x, in, sizeof x);
    for (int r = 0; r < 6; r++) {
        salsa_quarter(x, 0, 4, 8, 12);
        salsa_quarter(x, 5, 9, 13, 1);
        salsa_quarter(x, 10, 14, 2, 6);
        salsa_quarter(x, 15, 3, 7, 11);
        salsa_quarter(x, 0, 1, 2, 3);
        salsa_quarter(x, 5, 6, 7, 4);
        salsa_quarter(x, 10, 11, 8, 9);
        salsa_quarter(x, 15, 12, 13, 14);
    }
    return ((u128)(x[1] + in[1]) << 96) | ((u128)(x[2] + in[2]) << 64) |
           ((u128)(x[3] + in[3]) << 32) | (u128)(x[4] + in[4]);
}

static void chacha_quarter(uint32_t *x, int a, int b, int c, int d)
{
    x[a] += x[b]; x[d] = rotl32(x[d] ^ x[a], 16);
    x[c] += x[d]; x[b] = rotl32(x[b] ^ x[c], 12);
    x[a] += x[b]; x[d] = rotl32(x[d] ^ x[a], 8);
    x[c] += x[d]; x[b] = rotl32(x[b] ^ x[c], 7);
}

/* dpf_base/dpf.h:145-196: ChaCha core, 12 rounds, key words MSW first in
 * in[4..7], position in in[13]; output = words 4..7 (word 4 = MSW). */
static u128 prf_chacha20_12(u128 seed, uint32_t pos)
{
    uint32_t in[16] = { 0 }, x[16];
    in[0] = SIGMA[0]; in[1] = SIGMA[1]; in[2] = SIGMA[2]; in[3] = SIGMA[3];
    in[4] = (uint32_t)(seed >> 96);
    in[5] = (uint32_t)(seed >> 64);
    in[6] = (uint32_t)(seed >> 32);
    in[7] = (uint32_t)seed;
    in[13] = pos;
    memcpy(x, in, sizeof x);
    for (int r = 0; r < 6; r++) {
        chacha_quarter(x, 0, 4, 8, 12);
        chacha_quarter(x, 1, 5, 9, 13);
        chacha_quarter(x, 2, 6, 10, 14);
        chacha_quarter(x, 3, 7, 11, 15);
        chacha_quarter(x, 0, 5, 10, 15);
        chacha_quarter(x, 1, 6, 11, 12);
        chacha_quarter(x, 2, 7, 8, 13);
        chacha_quarter(x, 3, 4, 9, 14);
    }
    return ((u128)(x[4] + in[4]) << 96) | ((u128)(x[5] + in[5]) << 64) |
           ((u128)(x[6] + in[6]) << 32) | (u128)(x[7] + in[7]);
}

/* --- AES-128, byte oriented, FIPS-197 ----------------------------------- */
static uint8_t g_sbox[256];
static int g_sbox_ready;

static uint8_t gf_mul(uint8_t a, uint8_t b)
{
    uint8_t p = 0;
    for (int i = 0; i < 8; i++) {
        if (b & 1) p ^= a;
        uint8_t hi = a & 0x80;
        a = (uint8_t)(a << 1);
        if (hi) a ^= 0x1b;
        b >>= 1;
    }
    return p;
}

static void sbox_init(void)
{
    if (g_sbox_ready) return;
    for (int v = 0; v < 256; v++) {
        /* multiplicative inverse by exhaustive search (0 -> 0) */
        uint8_t inv = 0;
        if (v) for (int c = 1; c < 256; c++) if (gf_mul((uint8_t)v, (uint8_t)c) == 1) { inv = (uint8_t)c; break; }
        uint8_t s = inv, r = inv;
        for (int k = 0; k < 4; k++) { r = (uint8_t)((r << 1) | (r >> 7)); s ^= r; }
        g_sbox[v] = s ^ 0x63;
    }
    g_sbox_ready = 1;
}

static void aes128_expand(const uint8_t key[16], uint8_t rk[176])
{
    memcpy(rk, key, 16);
    uint8_t rcon = 1;
    for (int w = 4; w < 44; w++) {
        uint8_t t[4];
        memcpy(t, rk + 4 * (w - 1), 4);
        if (w % 4 == 0) {
            uint8_t t0 = t[0];
            t[0] = g_sbox[t[1]] ^ rcon; t[1] = g_sbox[t[2]]; t[2] = g_sbox[t[3]]; t[3] = g_sbox[t0];
            rcon = gf_mul(rcon, 2);
        }
        for (int k = 0; k < 4; k++) rk[4 * w + k] = rk[4 * (w - 4) + k] ^ t[k];
    }
}

void orc_aes128_encrypt(const uint8_t key[16], const uint8_t in[16], uint8_t out[16])
{
    sbox_init();
    uint8_t rk[176], s[16], t[16];
    aes128_expand(key, rk);
    for (int i = 0; i < 16; i++) s[i] = in[i] ^ rk[i];
    for (int round = 1; round <= 10; round++) {
        /* SubBytes + ShiftRows: byte (row r, col c) lives at s[4c + r] */
        for (int c = 0; c < 4; c++)
            for (int r = 0; r < 4; r++)
                t[4 * c + r] = g_sbox[s[4 * ((c + r) & 3) + r]];
        if (round < 10) {
            for (int c = 0; c < 4; c++) {
                uint8_t a0 = t[4 * c], a1 = t[4 * c + 1], a2 = t[4 * c + 2], a3 = t[4 * c + 3];
                s[4 * c + 0] = gf_mul(a0, 2) ^ gf_mul(a1, 3) ^ a2 ^ a3;
                s[4 * c + 1] = a0 ^ gf_mul(a1, 2) ^ gf_mul(a2, 3) ^ a3;
                s[4 * c + 2] = a0 ^ a1 ^ gf_mul(a2, 2) ^ gf_mul(a3, 3);
                s[4 * c + 3] = gf_mul(a0, 3) ^ a1 ^ a2 ^ gf_mul(a3, 2);
            }
        } else {
            memcpy(s, t, 16);
        }
        for (int i = 0; i < 16; i++) s[i] ^= rk[16 * round + i];
    }
    memcpy(out, s, 16);
}

/* dpf_base/dpf.h:198-219: AES-128 keyed by the 16 little-endian bytes of the
 * seed, encrypting the 16 little-endian bytes of the position. */
static u128 prf_aes128(u128 seed, uint32_t pos)
{
    uint8_t key[16], in[16] = { 0 }, out[16];
    u128 p = pos, r;
    memcpy(key, &seed, 16);
    memcpy(in, &p, 16);
    orc_aes128_encrypt(key, in, out);
    memcpy(&r, out, 16);
    return r;
}

/* dpf_base/dpf.h:226-235 (PRF_SELECT) */
static u128 prf_eval(int prf, u128 seed, uint32_t pos)
{
    switch (prf) {
    case ORC_PRF_DUMMY: return prf_dummy(seed, pos);
    case ORC_PRF_SALSA20: return prf_salsa20_12(seed, pos);
    case ORC_PRF_CHACHA20: return prf_chacha20_12(seed, pos);
    case ORC_PRF_AES128: return prf_aes128(seed, pos);
    default: abort();
    }
}

void orc_prf(int prf, uint64_t seed_lo, uint64_t seed_hi, uint32_t pos,
             uint64_t *out_lo, uint64_t *out_hi)
{
    u128 r = prf_eval(prf, mk128(seed_lo, seed_hi), pos);
    *out_lo = (uint64_t)r;
    *out_hi = (uint64_t)(r >> 64);
}

/* ------------------------------------------------------------------------ */
/* evaluation                                                                */
/* ------------------------------------------------------------------------ */

/* One tree step (dpf_base/dpf.h:368-374): the correction-word bank is picked
 * by the LSB of the PARENT seed; `level` counts depth-1 at the root down to 0
 * at the leaves and selects cw[2*level + bit]. */
static u128 step(const int32_t *key, int prf, u128 parent, int level, int bit)
{
    int bank = (parent & 1) ? SLOT_CW2 : SLOT_CW1;
    return prf_eval(prf, parent, (uint32_t)bit) + key_slot(key, bank + 2 * level + bit);
}

static u128 eval_flat(const int32_t *key, int64_t idx, int prf)
{
    int depth = (int)key_slot(key, SLOT_DEPTH);
    u128 s = key_slot(key, SLOT_ROOT);
    for (int level = depth - 1; level >= 0; level--) {
        s = step(key, prf, s, level, (int)(idx & 1));
        idx >>= 1;
    }
    return s;
}

void orc_eval_flat(const int32_t *key, int64_t idx, int prf,
                   uint64_t *out_lo, uint64_t *out_hi)
{
    u128 r = eval_flat(key, idx, prf);
    *out_lo = (uint64_t)r;
    *out_hi = (uint64_t)(r >> 64);
}

/* An early-terminated key (slot 0 = (d, 2, 0, 0)): the same walk over the d levels of leaf `leaf`,
 * except that the level-0 correction word is added lane-wise in (Z/2^32)^4 (DESIGN.md section 9). */
static void eval_flat_et(const int32_t *key, int64_t leaf, int prf, uint32_t out[4])
{
    int depth = key[0];
    u128 s = key_slot(key, SLOT_ROOT);
    for (int level = depth - 1; level >= 0; level--) {
        int bit = (int)(leaf & 1);
        int bank = (s & 1) ? SLOT_CW2 : SLOT_CW1;
        u128 v = prf_eval(prf, s, (uint32_t)bit), cw = key_slot(key, bank + 2 * level + bit);
        if (level > 0) {
            s = v + cw;
        } else {
            s = 0;
            for (int l = 0; l < 4; l++)
                s |= (u128)(uint32_t)((uint32_t)(v >> (32 * l)) + (uint32_t)(cw >> (32 * l))) << (32 * l);
        }
        leaf >>= 1;
    }
    for (int l = 0; l < 4; l++) out[l] = (uint32_t)(s >> (32 * l));
}

typedef struct {
    const int32_t *keys;
    int64_t nkeys, npoints;
    int prf, et, nthreads, t;
    const int64_t *points;
    int32_t *out;
} points_job;

static void *points_worker(void *arg)
{
    const points_job *j = (const points_job *)arg;
    const int64_t total = j->nkeys * j->npoints;
    for (int64_t w = j->t; w < total; w += j->nthreads) {
        const int32_t *key = j->keys + (w / j->npoints) * ORC_KEY_WORDS;
        const int64_t x = j->points[w % j->npoints];
        if (j->et) {
            eval_flat_et(key, x, j->prf, (uint32_t *)j->out + 4 * w);
        } else {
            j->out[w] = (int32_t)(uint32_t)eval_flat(key, x, j->prf);
        }
    }
    return NULL;
}

static int eval_points(const int32_t *keys, int64_t nkeys, int prf, const int64_t *points, int64_t npoints,
                       int nthreads, int et, int32_t *out)
{
    if (nkeys < 0 || npoints < 0 || prf < 0 || prf > 3) return -1;
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    sbox_init();   /* once, before the threads share it */
    pthread_t th[256];
    points_job jobs[256];
    int started = 0, rc = 0;
    for (int t = 0; t < nthreads; t++) {
        jobs[t] = (points_job){ keys, nkeys, npoints, prf, et, nthreads, t, points, out };
        if (t == 0) continue;
        if (pthread_create(&th[t], NULL, points_worker, &jobs[t]) != 0) { rc = -3; break; }
        started = t;
    }
    points_worker(&jobs[0]);
    for (int t = 1; t <= started; t++) pthread_join(th[t], NULL);
    if (rc) return rc;   /* some share of the work was never done */
    return 0;
}

int orc_eval_points(const int32_t *keys, int64_t nkeys, int prf, const int64_t *idx, int64_t nidx,
                    int nthreads, int32_t *out)
{
    return eval_points(keys, nkeys, prf, idx, nidx, nthreads, 0, out);
}

int orc_eval_points_et(const int32_t *keys, int64_t nkeys, int prf, const int64_t *leaves, int64_t nleaves,
                       int nthreads, int32_t *out)
{
    return eval_points(keys, nkeys, prf, leaves, nleaves, nthreads, 1, out);
}

int orc_eval_full_flat(const int32_t *key, int prf, int32_t *out_n)
{
    int64_t n = (int64_t)key_slot(key, SLOT_N);
    for (int64_t i = 0; i < n; i++) out_n[i] = (int32_t)(uint32_t)eval_flat(key, i, prf);
    return 0;
}

uint32_t orc_bitrev(uint32_t x, int bits)
{
    uint32_t r = 0;
    for (int i = 0; i < bits; i++) r |= ((x >> i) & 1u) << (bits - 1 - i);
    return r;
}

/* Level-by-level expansion.  After `k` levels, position p (k bits, first
 * consumed index bit = MSB of p) holds the seed of every index whose low k
 * bits are bitrev_k(p).  Returns the leaves in BFS position order. */
static u128 *expand_tree(const int32_t *key, int prf, int *depth_out)
{
    int depth = (int)key_slot(key, SLOT_DEPTH);
    int64_t n = (int64_t)1 << depth;
    u128 *cur = (u128 *)malloc(sizeof(u128) * (size_t)n);
    u128 *nxt = (u128 *)malloc(sizeof(u128) * (size_t)n);
    if (!cur || !nxt) { free(cur); free(nxt); return NULL; }
    cur[0] = key_slot(key, SLOT_ROOT);
    for (int k = 0; k < depth; k++) {
        int level = depth - 1 - k;
        int64_t width = (int64_t)1 << k;
        for (int64_t p = 0; p < width; p++) {
            nxt[2 * p] = step(key, prf, cur[p], level, 0);
            nxt[2 * p + 1] = step(key, prf, cur[p], level, 1);
        }
        u128 *t = cur; cur = nxt; nxt = t;
    }
    free(nxt);
    *depth_out = depth;
    return cur;
}

int orc_eval_full_tree(const int32_t *key, int prf, int32_t *out_n)
{
    int depth;
    u128 *leaves = expand_tree(key, prf, &depth);
    if (!leaves) return -1;
    int64_t n = (int64_t)1 << depth;
    for (int64_t p = 0; p < n; p++)
        out_n[orc_bitrev((uint32_t)p, depth)] = (int32_t)(uint32_t)leaves[p];
    free(leaves);
    return 0;
}

int orc_eval_dot(const int32_t *keys, int64_t nkeys, int prf,
                 const int32_t *table, int64_t n, int entry_size,
                 int use_tree, int32_t *out)
{
    int32_t *share = (int32_t *)malloc(sizeof(int32_t) * (size_t)n);
    if (!share) return -1;
    for (int64_t b = 0; b < nkeys; b++) {
        const int32_t *key = keys + b * ORC_KEY_WORDS;
        if ((int64_t)key_slot(key, SLOT_N) != n) { free(share); return -2; }
        int rc = use_tree ? orc_eval_full_tree(key, prf, share) : orc_eval_full_flat(key, prf, share);
        if (rc) { free(share); return rc; }
        for (int e = 0; e < entry_size; e++) {
            uint32_t acc = 0;
            for (int64_t i = 0; i < n; i++)
                acc += (uint32_t)share[i] * (uint32_t)table[i * entry_size + e];
            out[b * entry_size + e] = (int32_t)acc;
        }
    }
    return 0;
}

int orc_eval_dot_range(const int32_t *keys, int64_t nkeys, int prf,
                       const int32_t *table, int64_t n, int entry_size,
                       int64_t idx_begin, int64_t idx_count, int32_t *out)
{
    if (idx_begin < 0 || idx_begin + idx_count > n || entry_size > 1024) return -1;
    for (int64_t b = 0; b < nkeys; b++) {
        const int32_t *key = keys + b * ORC_KEY_WORDS;
        uint32_t acc[1024] = { 0 };
        for (int64_t i = idx_begin; i < idx_begin + idx_count; i++) {
            uint32_t share = (uint32_t)eval_flat(key, i, prf);
            for (int e = 0; e < entry_size; e++)
                acc[e] += share * (uint32_t)table[i * entry_size + e];
        }
        for (int e = 0; e < entry_size; e++) out[b * entry_size + e] = (int32_t)acc[e];
    }
    return 0;
}

int orc_eval_dot_shard(const int32_t *key, int prf, const int32_t *table,
                       int64_t n, int entry_size, int64_t pos_begin,
                       int64_t pos_count, int32_t *out)
{
    int depth;
    u128 *leaves = expand_tree(key, prf, &depth);
    if (!leaves) return -1;
    if (((int64_t)1 << depth) != n) { free(leaves); return -2; }
    for (int e = 0; e < entry_size; e++) {
        uint32_t acc = 0;
        for (int64_t p = pos_begin; p < pos_begin + pos_count; p++) {
            int64_t idx = orc_bitrev((uint32_t)p, depth);
            acc += (uint32_t)leaves[p] * (uint32_t)table[idx * entry_size + e];
        }
        out[e] = (int32_t)acc;
    }
    free(leaves);
    return 0;
}

/* ------------------------------------------------------------------------ */
/* key generation                                                            */
/* ------------------------------------------------------------------------ */

/* MT19937 (Matsumoto & Nishimura 1998), the engine behind std::mt19937 that
 * the reference seeds at dpf_wrapper.cu:52. */
typedef struct { uint32_t mt[624]; int idx; } mt19937_t;

static void mt_seed(mt19937_t *g, uint32_t s)
{
    g->mt[0] = s;
    for (int i = 1; i < 624; i++)
        g->mt[i] = 1812433253u * (g->mt[i - 1] ^ (g->mt[i - 1] >> 30)) + (uint32_t)i;
    g->idx = 624;
}

static uint32_t mt_next(mt19937_t *g)
{
    if (g->idx >= 624) {
        for (int i = 0; i < 624; i++) {
            uint32_t y = (g->mt[i] & 0x80000000u) | (g->mt[(i + 1) % 624] & 0x7fffffffu);
            g->mt[i] = g->mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        g->idx = 0;
    }
    uint32_t y = g->mt[g->idx++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

/* std::uniform_int_distribution<uint64_t>(0, 2^64-1) over a 32-bit engine as
 * libstdc++ composes it: high word drawn first, then the low word. */
static uint64_t rand64(mt19937_t *g)
{
    uint64_t hi = mt_next(g);
    uint64_t lo = mt_next(g);
    return (hi << 32) | lo;
}

/* dpf_base/dpf.h:272-277 (GenerateRandomNumber): first draw is the high half. */
static u128 rand128(mt19937_t *g)
{
    uint64_t l = rand64(g);
    uint64_t r = rand64(g);
    return ((u128)l << 64) | r;
}

/* dpf_base/dpf.h:279-283 */
static u128 rand128_odd(mt19937_t *g)
{
    u128 k = 0;
    while ((k & 1) == 0) k = rand128(g);
    return k;
}

/*
 * dpf_base/dpf.h:403-464 (log construction) with the N==2 base case of
 * dpf.h:290-360, flattened as dpf.h:239-270 and packed as dpf_wrapper.cu:26-35.
 *
 * The reference recurses from the full domain down to N=2, drawing one odd
 * "beta" per level on the way down, then builds correction words on the way
 * back up.  Here the same draws are made by a down loop and an up loop.
 * Flat level L (0 = full domain ... depth-1 = the N=2 base) owns cw[2L], cw[2L+1].
 */
int orc_gen(int64_t alpha, int64_t n, uint32_t seed32, int prf,
            int32_t *key_a, int32_t *key_b)
{
    if (n < 2 || (n & (n - 1)) || alpha < 0 || alpha >= n) return -1;
    int depth = 0;
    while (((int64_t)1 << depth) < n) depth++;
    if (depth > 32) return -1;

    mt19937_t g;
    mt_seed(&g, seed32);

    u128 beta[33];
    beta[0] = 1;                                   /* dpf_wrapper.cu:53: beta = 1 */
    for (int L = 0; L < depth - 1; L++) beta[L + 1] = rand128_odd(&g);

    u128 cw1[64] = { 0 }, cw2[64] = { 0 };

    /* base level (domain of 2, one seed per server) */
    int base = depth - 1;
    int a_base = (int)(alpha & 1);                 /* target row at the base */
    u128 k1 = rand128(&g), k2 = rand128(&g);
    k1 &= ~(u128)1;
    k2 = (k2 & ~(u128)1) | 1;
    u128 diff[2];
    for (int i = 0; i < 2; i++) {
        diff[i] = prf_eval(prf, k1, (uint32_t)i) - prf_eval(prf, k2, (uint32_t)i);
        if (i == a_base) diff[i] -= beta[base];
    }
    for (int i = 0; i < 2; i++) {
        cw1[2 * base + i] = rand128(&g);
        cw2[2 * base + i] = cw1[2 * base + i] + diff[i];
    }
    /* seeds of the two servers on the alpha path after the base level */
    u128 s1 = prf_eval(prf, k1, (uint32_t)a_base) + ((k1 & 1) ? cw2 : cw1)[2 * base + a_base];
    u128 s2 = prf_eval(prf, k2, (uint32_t)a_base) + ((k2 & 1) ? cw2 : cw1)[2 * base + a_base];

    for (int L = depth - 2; L >= 0; L--) {
        int row = (int)((alpha >> (depth - 1 - L)) & 1);   /* alpha_L / (N_L/2) */
        for (int i = 0; i < 2; i++) {
            u128 d = prf_eval(prf, s2, (uint32_t)i) - prf_eval(prf, s1, (uint32_t)i);
            if ((s1 & 1) == 0) d = (u128)0 - d;
            cw1[2 * L + i] = (u128)mt_next(&g);
            cw2[2 * L + i] = cw1[2 * L + i] + d;
            if (i == row) {
                if ((s1 & 1) == 0) cw1[2 * L + i] += beta[L];
                else cw1[2 * L + i] -= beta[L];
            }
        }
        u128 n1 = prf_eval(prf, s1, (uint32_t)row) + ((s1 & 1) ? cw2 : cw1)[2 * L + row];
        u128 n2 = prf_eval(prf, s2, (uint32_t)row) + ((s2 & 1) ? cw2 : cw1)[2 * L + row];
        s1 = n1; s2 = n2;
    }

    memset(key_a, 0, sizeof(int32_t) * ORC_KEY_WORDS);
    memset(key_b, 0, sizeof(int32_t) * ORC_KEY_WORDS);
    key_set_slot(key_a, SLOT_DEPTH, (u128)depth);
    key_set_slot(key_b, SLOT_DEPTH, (u128)depth);
    for (int i = 0; i < 64; i++) {
        key_set_slot(key_a, SLOT_CW1 + i, cw1[i]); key_set_slot(key_b, SLOT_CW1 + i, cw1[i]);
        key_set_slot(key_a, SLOT_CW2 + i, cw2[i]); key_set_slot(key_b, SLOT_CW2 + i, cw2[i]);
    }
    key_set_slot(key_a, SLOT_ROOT, k1);
    key_set_slot(key_b, SLOT_ROOT, k2);
    key_set_slot(key_a, SLOT_N, (u128)n);
    key_set_slot(key_b, SLOT_N, (u128)n);
    return 0;
}
