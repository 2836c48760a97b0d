/*
 * oracle/dpf_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C CPU restatement of the reference algorithm for the one hot path
 * (batched full-domain evaluation of log(n)-key DPFs fused with the int32
 * inner product).  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load this library.  The product
 * (gpu-dpf_b200/) never links, imports or calls it.
 *
 * Parity status: PINNED.  Every function here is checked against the real
 * reference (dpf_base/dpf.h compiled unmodified into oracle/_ref/libdpfref.so
 * by oracle/Makefile) in tests/test_oracle_vs_ref.py, and against the golden
 * vectors generated from that build in tests/golden/.
 *
 * Each function cites the reference file:line it restates (paths relative to
 * the reference repository root).
 */
#ifndef DPF_ORACLE_H
#define DPF_ORACLE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef unsigned __int128 u128;

/* PRF ids: dpf_base/dpf.h:221-224, dpf_wrapper.cu:200-203 */
enum { ORC_PRF_DUMMY = 0, ORC_PRF_SALSA20 = 1, ORC_PRF_CHACHA20 = 2, ORC_PRF_AES128 = 3 };

/* One server's key on the wire: int32[524] == 131 little-endian u128 slots
 * (dpf_wrapper.cu:26-46): [0]=depth, [1..64]=cw_1, [65..128]=cw_2,
 * [129]=root seed, [130]=n. */
#define ORC_KEY_WORDS 524

/* 128-bit value <-> two u64 halves (lo, hi) so ctypes can talk to us. */
void orc_prf(int prf, uint64_t seed_lo, uint64_t seed_hi, uint32_t pos,
             uint64_t *out_lo, uint64_t *out_hi);

/* AES-128 single-block encrypt (FIPS-197), for the C.1 known-answer test. */
void orc_aes128_encrypt(const uint8_t key[16], const uint8_t in[16], uint8_t out[16]);

/* dpf_base/dpf.h:362-377 (EvaluateFlat): value at one index, full 128 bits. */
void orc_eval_flat(const int32_t *key, int64_t idx, int prf,
                   uint64_t *out_lo, uint64_t *out_hi);

/* Batched per-index walks for sparse checks at any n: out[b][j] = low32(EvaluateFlat(keys[b], idx[j]))
 * for nkeys keys (int32[nkeys][524]) and nidx indices, spread over `nthreads` host threads.  Each value
 * is one root-to-leaf walk (the loop of orc_eval_flat), so the cost is O(nkeys * nidx * depth),
 * independent of n.  Returns 0, or a negative code (bad argument, a thread that could not start). */
int orc_eval_points(const int32_t *keys, int64_t nkeys, int prf, const int64_t *idx, int64_t nidx,
                    int nthreads, int32_t *out);

/* The same for early-terminated keys (slot 0 = (d, 2, 0, 0); DESIGN.md section 9): out[b][j][0..3] =
 * the four 32-bit words of leaf leaves[j], i.e. the shares of rows 4*leaves[j] .. 4*leaves[j]+3.  Not
 * pinned against the reference, which has no such keys; tests/et_oracle.py states the same walk. */
int orc_eval_points_et(const int32_t *keys, int64_t nkeys, int prf, const int64_t *leaves, int64_t nleaves,
                       int nthreads, int32_t *out);

/* dpf_wrapper.cu:70-84 (eval_dpf_cpu): low 32 bits of EvaluateFlat for every
 * index, natural order, via per-index root-to-leaf walks (n*log n PRFs). */
int orc_eval_full_flat(const int32_t *key, int prf, int32_t *out_n);

/* Same values through one GGM tree expansion (2n-2 PRFs); used for big n. */
int orc_eval_full_tree(const int32_t *key, int prf, int32_t *out_n);

/* dpf.py:85-86 + dpf_wrapper.cu:178-185: out[b][e] = sum_i share_b[i]*table[i][e]
 * mod 2^32 for a batch of keys; table is int32 [n][E] row-major, natural
 * index order.  use_tree selects orc_eval_full_tree over the per-index walk. */
int orc_eval_dot(const int32_t *keys, int64_t nkeys, int prf,
                 const int32_t *table, int64_t n, int entry_size,
                 int use_tree, int32_t *out);

/* Bounded-sample form of the per-index reference path, for CPU-baseline timing:
 * the inner product restricted to natural indices [idx_begin, idx_begin+idx_count)
 * using one EvaluateFlat walk per index (dpf_base/dpf.h:362-377). */
int orc_eval_dot_range(const int32_t *keys, int64_t nkeys, int prf,
                       const int32_t *table, int64_t n, int entry_size,
                       int64_t idx_begin, int64_t idx_count, int32_t *out);

/* Partial sum over the BFS leaf positions [pos_begin, pos_begin+pos_count) --
 * the entry-range shard of SURVEY.md section 8(e).  Leaf position p holds
 * index bitrev_depth(p). */
int orc_eval_dot_shard(const int32_t *key, int prf, const int32_t *table,
                       int64_t n, int entry_size, int64_t pos_begin,
                       int64_t pos_count, int32_t *out);

/* dpf_wrapper.cu:49-68 (gen) -> dpf_base/dpf.h:403-464, 290-360, 239-270:
 * two-server key generation, beta = 1, std::mt19937 seeded with the low 32
 * bits of `seed32`. */
int orc_gen(int64_t alpha, int64_t n, uint32_t seed32, int prf,
            int32_t *key_a, int32_t *key_b);

/* bit reversal of the low `bits` bits (dpf_gpu/utils.h:142-149 + dpf_wrapper.cu:106). */
uint32_t orc_bitrev(uint32_t x, int bits);

#ifdef __cplusplus
}
#endif
#endif
