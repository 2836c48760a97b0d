/*
 * dpf_host.h -- host-side (CPU) parts of the engine's API: the key wire format,
 * client key generation and the API's CPU evaluation function.  These mirror
 * CPU-only entry points of the reference extension (dpf_wrapper.cu:26-84); the
 * GPU path never routes through them.
 */
#pragma once

#include <stdint.h>

#include "dpf_core.cuh"

namespace b200dpf {
namespace host {

/* wire format, dpf_wrapper.cu:26-46: 131 little-endian 128-bit slots */
enum : int { KEY_WORDS = 524, SLOT_DEPTH = 0, SLOT_CW1 = 1, SLOT_CW2 = 65, SLOT_ROOT = 129, SLOT_N = 130 };

/* Te0 in the little-endian column convention of dpf_core.cuh (256 words),
 * built once from a computed S-box. */
const uint32_t *aes_te0();
/* The AES S-box (256 bytes). */
const uint8_t *aes_sbox();

Seed prf(int prf_id, const Seed &s, uint32_t pos);

inline Seed key_slot(const int32_t *key, int slot)
{
    const uint32_t *p = reinterpret_cast<const uint32_t *>(key) + 4 * slot;
    return make_seed(p[0], p[1], p[2], p[3]);
}

/* The kinds of key.  A key of every kind is a tree of 2^depth leaves over n = 2^(depth + lane_bits) table
 * rows, slot 0 = (depth, lane_bits, 0, 0), slot 130 = n as a u64; a leaf carries 2^lane_bits row shares:
 *   standard          one row per leaf, level 0 in Z/2^128 (the reference's keys)
 *   early-terminated  four rows per leaf, level 0 in (Z/2^32)^4 (DESIGN.md section 9)
 *   XOR-shared        128 one-bit row shares per leaf, level 0 in (Z/2)^128; row i is bit (i & 127) of
 *                     leaf i >> 7, and the results XOR instead of adding (section 10) */
enum KeyKind : int { KIND_STANDARD = 0, KIND_ET = 1, KIND_XOR = 2, KIND_COUNT = 3 };

struct KindInfo {
    int lane_bits;          /* log2 table rows per leaf */
    int max_depth;
    int64_t n_min, n_max;   /* of the keys gen_leaves / gen make */
    char magic[5];          /* of the compact form (b200dpf_key_pack) */
    int group;              /* of level 0, dpf_core.cuh */
    const char *name;       /* in messages */
};

constexpr KindInfo kKinds[KIND_COUNT] = {
    {0, 32, 2, (int64_t)1 << 32, "DPF2", GROUP_ADD128, "standard"},
    {2, 29, 8, (int64_t)1 << 31, "DPE4", GROUP_LANES32, "early-terminated"},
    {7, 24, 256, (int64_t)1 << 31, "DPX7", GROUP_XOR128, "XOR-shared"},
};

/* The depth (1..max_depth) or n of a well-formed key of `kind`, or -1 for anything else -- a key of
 * another kind included.  key_depth reads slot 0 only. */
int key_depth(const int32_t *key, int kind);
int64_t key_n(const int32_t *key, int kind);
/* the kind of a well-formed key, or -1 */
int key_kind(const int32_t *key);

/* standard keys: the reference's mt19937 generator seeded with 32 bits, or (gen_secure) the ChaCha20
 * DRBG with key = seed[0..31], nonce = seed[32..43] */
int gen(int64_t alpha, int64_t n, uint32_t seed32, int prf_id, int32_t *key_a, int32_t *key_b);
int gen_secure(int64_t alpha, int64_t n, const uint8_t seed[44], int prf_id, int32_t *key_a, int32_t *key_b);
/* early-terminated or XOR-shared key for row alpha of an n-row table (n_min <= n <= n_max, a power of
 * two), drawn from the ChaCha20 DRBG like gen_secure */
int gen_leaves(int kind, int64_t alpha, int64_t n, const uint8_t seed[44], int prf_id, int32_t *key_a, int32_t *key_b);
/* The key's share of all n rows: int32 [n], or for XOR-shared keys the share bits packed, uint32 [n / 32]
 * in natural order (row i = bit i & 31 of word i >> 5).  -1 for a key that is not of `kind` (or a
 * standard key deeper than 31), -2 for an unknown prf id. */
int eval_cpu(const int32_t *key, int kind, int prf_id, int32_t *out);

}  // namespace host
}  // namespace b200dpf
