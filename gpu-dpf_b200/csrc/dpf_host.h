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

/* depth / n sanity: returns depth (1..32) or -1 */
int key_depth(const int32_t *key);
int64_t key_n(const int32_t *key);

/* Early-terminated keys (DESIGN.md section 9): a tree of 2^depth leaves over n = 4 * 2^depth
 * table rows, slot 0 = (depth, 2, 0, 0), slot 130 = n.  These return the tree depth (1..29)
 * or n, or -1 for anything else -- a standard key included. */
enum : int { ET_LOG2_ROWS_PER_LEAF = 2, ET_MAX_DEPTH = 29 };
int key_et_depth(const int32_t *key);
int64_t key_et_n(const int32_t *key);

int gen(int64_t alpha, int64_t n, uint32_t seed32, int prf_id, int32_t *key_a, int32_t *key_b);
/* ChaCha20-DRBG variant: key = seed[0..31], nonce = seed[32..43] */
int gen_secure(int64_t alpha, int64_t n, const uint8_t seed[44], int prf_id, int32_t *key_a, int32_t *key_b);
int eval_cpu(const int32_t *key, int prf_id, int32_t *out_n);
/* Early-terminated key for row alpha of an n-row table (8 <= n <= 2^31, a power of two), drawn
 * from the ChaCha20 DRBG like gen_secure; eval_cpu_et writes its share of all n rows. */
int gen_et(int64_t alpha, int64_t n, const uint8_t seed[44], int prf_id, int32_t *key_a, int32_t *key_b);
int eval_cpu_et(const int32_t *key, int prf_id, int32_t *out_n);

/* XOR-shared keys (DESIGN.md section 10): a tree of 2^depth leaves over n = 128 * 2^depth table rows,
 * slot 0 = (depth, 7, 0, 0), slot 130 = n; row i is bit (i & 127) of leaf i >> 7.  The checks return
 * the tree depth (1..24) or n, or -1 for anything else -- a standard or early-terminated key included. */
enum : int { XOR_LOG2_ROWS_PER_LEAF = 7, XOR_MAX_DEPTH = 24 };
int key_xor_depth(const int32_t *key);
int64_t key_xor_n(const int32_t *key);
/* Key for row alpha of an n-row table (256 <= n <= 2^31, a power of two), drawn from the ChaCha20 DRBG;
 * eval_cpu_xor writes its share bits packed, bits[n / 32] in natural order (row i = bit i & 31 of
 * word i >> 5). */
int gen_xor(int64_t alpha, int64_t n, const uint8_t seed[44], int prf_id, int32_t *key_a, int32_t *key_b);
int eval_cpu_xor(const int32_t *key, int prf_id, uint32_t *bits);

}  // namespace host
}  // namespace b200dpf
