/*
 * b200dpf.h -- C ABI of the H100-native DPF evaluation engine.
 *
 * This is the drop-in boundary for the ONE hot path of facebookresearch/GPU-DPF:
 * batched full-domain evaluation of log(n)-key distributed point functions
 * fused with the int32 inner product against the server's table.  Everything a
 * binding of that path needs is here as plain pointers and sizes (no torch, no
 * C++ types).  The reference reaches the same functionality through the five
 * pybind functions of dpf_wrapper.cu:188-204; each entry point below names the
 * reference interface it stands in for.
 *
 * Conventions
 *   - every function returns 0 on success, a negative B200DPF_E* code on
 *     failure; b200dpf_last_error() returns a thread-local message.
 *   - a key is the reference's wire format: int32[524] == 131 little-endian
 *     128-bit slots, [0]=depth, [1..64]=cw_1, [65..128]=cw_2, [129]=root seed,
 *     [130]=n                                  (dpf_wrapper.cu:26-46).
 *   - PRF ids are the reference's: 0 DUMMY, 1 SALSA20, 2 CHACHA20, 3 AES128
 *                                              (dpf_wrapper.cu:200-203).
 *   - results: out[b][e] = int32( sum_i low32(EvaluateFlat(key_b, i)) *
 *     uint32(table[i][e]) mod 2^32 )           (dpf_base/dpf.h:362-377 +
 *     dpf_wrapper.cu:178-185 + dpf.py:85-86).
 *
 * The GPU entry points require a CUDA device and fail with B200DPF_ECUDA when
 * none is usable: there is no CPU fallback behind them.
 *
 * Threading: a context is NOT re-entrant -- its device scratch (ticket counters, frontier,
 * leaf cache, key/result staging) serves one evaluation at a time, so calls on one context must
 * come from one host thread at a time.  Evaluations enqueued on DIFFERENT streams through the
 * *_device entry points are ordered by the library (each waits for the context's previous
 * evaluation).  Use one context per concurrent stream of work; contexts are independent.
 * Tested (tests/test_gpu_concurrency.py, tests/test_concurrency_host.py): independent contexts of
 * every kind, plain, trimmed and grouped, used from any host threads of one device at once, while
 * other threads create and destroy contexts and generate keys; one context used by several threads
 * in turn, each enqueueing on its own stream without synchronising before it hands over; and the
 * ordering across streams, including calls whose larger batches grow the context's scratch while
 * earlier calls may still run, row updates and accumulating calls.  The host entry points (key
 * generation, host evaluation, key packing) may be called from any number of threads, and
 * b200dpf_last_error reports the calling thread's last failure.
 */
#ifndef B200DPF_H
#define B200DPF_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200DPF_KEY_WORDS 524          /* int32 words per key (2096 bytes)      */
#define B200DPF_DEFAULT_ENTRY_SIZE 16  /* dpf_wrapper.cu:18  (MM)               */
#define B200DPF_DEFAULT_BATCH_SIZE 512 /* dpf_wrapper.cu:21  (BATCH_SIZE)       */

enum {
    B200DPF_PRF_DUMMY = 0,
    B200DPF_PRF_SALSA20 = 1,
    B200DPF_PRF_CHACHA20 = 2,
    B200DPF_PRF_AES128 = 3
};

enum {
    B200DPF_OK = 0,
    B200DPF_EINVAL = -1,   /* bad argument (shape, power of two, prf id, ...)   */
    B200DPF_ECUDA = -2,    /* CUDA runtime error or no usable device            */
    B200DPF_ENOMEM = -3,
    B200DPF_ESTATE = -4,   /* call out of order (e.g. eval before table upload) */
    B200DPF_EFULL = -5     /* a keyword-PIR placement did not finish (b200dpf_kwpir_create) */
};

typedef struct b200dpf_ctx b200dpf_ctx;

/* Library identification: "b200dpf <semver> sm_90a". */
const char *b200dpf_version(void);

/* Thread-local description of the last failure on this thread. */
const char *b200dpf_last_error(void);

/* ------------------------------------------------------------------------- */
/* Client side (CPU).                                                         */
/* ------------------------------------------------------------------------- */

/*
 * Two-server key generation for the point function f(alpha) = 1.
 * Replaces: dpf_cpp.gen -> gen()                          dpf_wrapper.cu:49-68
 *           (GenerateSeedsAndCodewordsLog dpf_base/dpf.h:403-464, FlattenCodewords :239-270).
 * `seed`/`seed_len`: the caller's entropy; like the reference, the generator is
 * std::mt19937 seeded with the first 4 bytes (little endian), so identical
 * seeds give keys identical to the reference's.
 * key_a/key_b: caller-allocated int32[524] each.
 */
int b200dpf_gen(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len,
                int prf, int32_t *key_a, int32_t *key_b);

/*
 * Key generation from a cryptographic generator (SURVEY.md section 8(f) rank 1; the
 * reference's own TODO at dpf.py:65 "replace with secure 128-bit RNG").  Same DPF
 * construction and wire format, but every random draw -- including the upper-level
 * correction words, which the reference draws as 32-bit values (dpf_base/dpf.h:450) --
 * is 128 bits of a ChaCha20 (RFC 8439) keystream keyed with seed[0..31] and nonce
 * seed[32..43].  seed_len must be >= 44 bytes of caller entropy.  Keys differ from
 * b200dpf_gen's for the same seed; they evaluate with the same entry points.
 */
int b200dpf_gen_secure(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len,
                       int prf, int32_t *key_a, int32_t *key_b);

/*
 * Batched key generation (SURVEY.md section 8(f) rank 1): `count` independent
 * b200dpf_gen calls spread over `nthreads` host threads (0 = all cores).
 * alphas[count]; seeds32[count] (one 32-bit generator seed per key);
 * keys_a/keys_b: int32[count][524].
 */
int b200dpf_gen_batch(const int64_t *alphas, const uint32_t *seeds32, int64_t count,
                      int64_t n, int prf, int nthreads,
                      int32_t *keys_a, int32_t *keys_b);

/* Batched b200dpf_gen_secure: seeds44 = count x 44 bytes of caller entropy (key || nonce per key). */
int b200dpf_gen_batch_secure(const int64_t *alphas, const uint8_t *seeds44, int64_t count,
                             int64_t n, int prf, int nthreads,
                             int32_t *keys_a, int32_t *keys_b);

/*
 * The same batched keygen on a GPU (one thread per key pair; SURVEY.md section 8(f) rank 1, "optionally
 * GPU"): bit-identical to b200dpf_gen_batch_secure for identical seeds.  alphas and seeds44 are host
 * arrays; keys_a / keys_b may be host or device memory ([count][524] int32), so a load generator can
 * leave the keys on the device and hand them to b200dpf_eval_device.  Key generation is the CLIENT's
 * step of the protocol; this entry point exists for benchmarks and load generators.
 */
int b200dpf_gen_batch_gpu(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                          int device, int32_t *keys_a, int32_t *keys_b);

/*
 * One server's share vector on the CPU, natural index order: out[i] =
 * (int32) low32(EvaluateFlat(key, i)), i < n (n read from the key).
 * Replaces: dpf_cpp.eval_cpu -> eval_dpf_cpu()            dpf_wrapper.cu:70-84.
 * This is the API's CPU function, not a fallback for the GPU path.
 */
int b200dpf_eval_cpu(const int32_t *key, int prf, int32_t *out_n);

/*
 * Compact wire form of a key (SURVEY.md section 8(f) rank 3).  Of the 131 slots of the
 * reference format only 4*depth correction words, the root seed and the depth are live
 * (dpf_base/dpf.h:18-29 sizes the arrays for n = 2^32).  Packed layout, little endian,
 * every field 16-byte aligned so the GPU reads it in place (b200dpf_eval_packed):
 *   "DPF2" | depth (u8) | 11 zero bytes | root seed (16) | per level L = 0..depth-1:
 *   cw_1[2L], cw_1[2L+1], cw_2[2L], cw_2[2L+1] (16 bytes each)
 * = 32 + 64*depth bytes (1312 at n = 2^20, 928 at n = 2^14, instead of 2096).  unpack()
 * restores the exact int32[524] key (unused slots zero), so packed keys evaluate
 * bit-identically.
 */
size_t b200dpf_key_packed_size(int depth);
int b200dpf_key_pack(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written);
int b200dpf_key_unpack(const uint8_t *in, size_t in_len, int32_t *key);

/* n stored in a key (slot 130) and its depth (slot 0); -1 if malformed. */
int64_t b200dpf_key_n(const int32_t *key);
int b200dpf_key_depth(const int32_t *key);

/* ------------------------------------------------------------------------- */
/* Server side (GPU, sm_90a).                                                 */
/* ------------------------------------------------------------------------- */

/*
 * Upload a table and build an evaluation context on CUDA device `device`.
 * Replaces: dpf_cpp.eval_init -> eval_init()              dpf_wrapper.cu:93-132
 *           (+ dpf_hybrid_initialize dpf_gpu/dpf/dpf_hybrid.cu:30-36).
 *
 * table:        int32 [n][entry_size] row-major, natural index order, host or
 *               device memory (any pointer cudaMemcpy can read).
 * n:            power of two, 2 <= n <= 2^31.
 * entry_size:   1 .. 4096 int32 columns (the reference fixes 16).
 * shard_rank / shard_count: entry-range sharding (SURVEY.md section 8(e)).
 *               shard_count must be a power of two <= n/2; this context then owns
 *               the GGM subtree under the depth-log2(shard_count) node with
 *               breadth-first index shard_rank, copies only those n/shard_count
 *               rows, and b200dpf_eval* returns PARTIAL sums that the caller
 *               adds (mod 2^32) across shards.  Pass (0, 1) for a whole table.
 */
int b200dpf_create(b200dpf_ctx **ctx, const int32_t *table, int64_t n, int entry_size,
                   int device, int shard_rank, int shard_count);

/*
 * One table on SEVERAL GPUs of this process (SURVEY.md section 8(b)/(e); the reference is
 * single-GPU: device 0 implicitly, dpf_wrapper.cu:114-129).  The returned context is used with
 * b200dpf_eval / b200dpf_eval_packed / b200dpf_destroy exactly like a single-device one, so a
 * caller of the reference API scales without a process launcher.
 *   axis B200DPF_AXIS_ENTRIES  device d owns entry-range shard (d, ndev) (ndev a power of two):
 *                              every device evaluates every key over its subtree and device
 *                              devices[0] adds the [nkeys][entry_size] partials with a kernel that
 *                              loads the peers' buffers over NVLink.
 *        B200DPF_AXIS_KEYS     every device holds the whole table and evaluates a contiguous
 *                              slice of the batch; nothing crosses GPUs.
 *        B200DPF_AXIS_AUTO     KEYS for n <= B200DPF_AUTO_KEYS_MAX_N (a shard of a small table
 *                              cannot keep a GPU busy), else ENTRIES.
 * One host thread per extra device issues that device's copies and launches.
 */
enum { B200DPF_AXIS_AUTO = 0, B200DPF_AXIS_ENTRIES = 1, B200DPF_AXIS_KEYS = 2 };
#define B200DPF_AUTO_KEYS_MAX_N (1 << 18)
int b200dpf_create_multi(b200dpf_ctx **ctx, const int32_t *table, int64_t n, int entry_size,
                         const int *devices, int ndev, int axis);

/* Devices behind a context (1 unless it came from b200dpf_create_multi) and its axis. */
int b200dpf_ctx_device_count(const b200dpf_ctx *ctx);
int b200dpf_ctx_axis(const b200dpf_ctx *ctx);

/*
 * Grouped evaluation -- the batch-PIR front end (SURVEY.md section 8(f) rank 4; the reference only
 * models it analytically: paper/experimental/batch_pir/batch_pir_optimization.py:84-87 charges one
 * DPF over every bin per query, :210-218 sums them).  One context holds `nbins` tables ("bins") of
 * possibly different power-of-two sizes n[g] (same entry_size); b200dpf_group_eval evaluates a mixed
 * list of (bin, key) pairs -- key b against table bins[b] -- in ONE launch: keys are sorted by bin,
 * cut into groups of <= 32 keys of one bin, and the work items of all groups form one ticket space,
 * so many small bins fill the GPU the way one big table does.
 *   out[b][e] = the same inner product b200dpf_eval would give for key b on table bins[b].
 * tables[g]: int32 [n[g]][entry_size], host or device.  keys: int32[nkeys][524]; bins: int32[nkeys].
 * b200dpf_group_create_et makes the same context for early-terminated keys (b200dpf_gen_et, see
 * below): every n[g] a power of two in [8, 2^31], each bin laid out as by b200dpf_create_et.  There
 * b200dpf_group_eval takes only keys of b200dpf_gen_et for n[bins[b]] rows (a standard key is EINVAL
 * before anything is copied), out[b][e] is what b200dpf_eval on b200dpf_create_et(table bins[b]) gives,
 * b200dpf_group_update_rows works as on a standard grouped context and b200dpf_ctx_rows_per_leaf is 4.
 * b200dpf_group_create_xor makes it for XOR-shared keys (b200dpf_gen_xor, see below): every n[g] a
 * power of two in [256, 2^31], each bin laid out as by b200dpf_create_xor.  There b200dpf_group_eval
 * takes only keys of b200dpf_gen_xor for n[bins[b]] rows (any other key is EINVAL before anything is
 * copied), out[b][e] is what b200dpf_eval on b200dpf_create_xor(table bins[b]) gives -- an XOR, so
 * out_a[b] ^ out_b[b] == table bins[b][alpha] --, b200dpf_group_update_rows works as on the other grouped
 * contexts and b200dpf_ctx_rows_per_leaf is 128.  Each grouped context refuses keys of the other two
 * kinds (EINVAL).
 */
int b200dpf_group_create(b200dpf_ctx **ctx, const int32_t *const *tables, const int64_t *n, int nbins,
                         int entry_size, int device);
int b200dpf_group_create_et(b200dpf_ctx **ctx, const int32_t *const *tables, const int64_t *n, int nbins,
                            int entry_size, int device);
int b200dpf_group_create_xor(b200dpf_ctx **ctx, const int32_t *const *tables, const int64_t *n, int nbins,
                             int entry_size, int device);
int b200dpf_group_eval(b200dpf_ctx *ctx, const int32_t *keys, const int32_t *bins, int64_t nkeys, int prf,
                       int32_t *out);

/*
 * Device-resident grouped evaluation: the computation of b200dpf_group_eval with keys and results in
 * device memory on the context's GPU, enqueued on `cuda_stream` (a cudaStream_t; NULL is the default
 * stream) with no host synchronisation, on every kind of grouped context.
 *   keys_dev: int32 [nkeys][524] (16-byte aligned), the wire format b200dpf_eval_device takes.
 *   bins:     int32 [nkeys] in HOST memory.  How many keys each bin has shapes the launch (key groups,
 *             work-item size, descriptors), so the host plans from the bins; reading them from the device
 *             would need a synchronisation.  In batch PIR the bin of each key is the layout of the query
 *             batch, which the server knows without reading the keys.
 *   out_dev:  int32 [nkeys][entry_size] (4-byte aligned).  out_dev[b] is bit for bit what
 *             b200dpf_group_eval returns for key b: sums mod 2^32 on standard and early-terminated
 *             contexts, XORs on XOR-shared ones.
 * The arguments are checked as by b200dpf_group_eval, before anything is enqueued: a context that is
 * not grouped is ESTATE; a null buffer, nkeys outside [1, 2^24], an unknown prf, a misaligned buffer or a
 * bin id outside [0, nbins) is EINVAL.  The keys themselves are NOT validated (as on b200dpf_eval_device):
 * a key's own header is never used to size or index anything -- its depth comes from its bin -- so a
 * malformed or wrong-kind key gives a meaningless result for that key, and nothing is read beyond its
 * 2096 bytes and its bin's table.  Both buffers must stay valid until the stream reaches the end of the
 * evaluation.
 * Ordering: the call joins the context's one-operation-in-flight chain (see "Threading" above), so it is
 * ordered against earlier and later b200dpf_group_eval, b200dpf_group_eval_device and
 * b200dpf_group_update_rows calls on any stream.
 * Host staging: the sort order, descriptors and work units go up from pinned buffers the context reuses
 * (b200dpf_group_eval plans into them too). A call never waits for its own work, but before it rewrites that
 * staging it waits on the host until the PREVIOUS b200dpf_group_eval_device call's uploads (not its kernels)
 * have run; b200dpf_group_eval waits for them the same way.
 * b200dpf_ctx_last_device_ms times the evaluation launches only (as for b200dpf_group_eval: the key gather
 * and result scatter are outside), and b200dpf_ctx_last_launches counts them.
 */
int b200dpf_group_eval_device(b200dpf_ctx *ctx, const void *keys_dev, const int32_t *bins, int64_t nkeys, int prf,
                              void *out_dev, void *cuda_stream);

/*
 * b200dpf_group_eval_device with the bin list in device memory too, planned on the GPU, for any mix of (bin, key)
 * pairs on every kind of grouped context, trimmed ones included.
 *   keys_dev: int32 [nkeys][524] (16-byte aligned), as for b200dpf_group_eval_device.
 *   bins_dev: int32 [nkeys] in device memory (4-byte aligned): key b is evaluated on bin bins_dev[b].
 *   out_dev:  int32 [nkeys][entry_size] (4-byte aligned).  out_dev[b] is bit for bit what b200dpf_group_eval_device
 *             returns for key b with the same bins on the host.  A key whose bin is outside [0, nbins) gets a zero
 *             row; the other keys' rows do not change.
 *   bad_dev:  NULL, or int64 in device memory (8-byte aligned) that receives the number of keys whose bin is out of
 *             range (written, not accumulated).
 * The arguments are checked as by b200dpf_group_eval_device, before anything is enqueued: a context that is not
 * grouped is ESTATE; a null buffer, nkeys outside [1, 2^24], an unknown prf or a misaligned buffer is EINVAL.  The
 * bin ids are not checked on the host (they are never read there), and the keys are not validated: a key's depth
 * comes from its bin.  Every buffer must stay valid until the stream reaches the end of the evaluation.
 * No host wait: the call enqueues everything on cuda_stream and returns.  The sort by bin, the key groups, their
 * work-item sizes, descriptors and work units, and the order list are computed on the device, into lists only this
 * entry point uses; the host does work that does not grow with nkeys.  The only exception is device scratch that
 * grows (an allocation) when nkeys grows past every earlier call's.  The host half of the plan is kept while nkeys,
 * prf and the context's options (b200dpf_ctx_set_option, b200dpf_ctx_set_subtree_log2) stay those of its previous call.
 * Ordering: the call joins the context's one-operation-in-flight chain (see "Threading" above), so it is ordered
 * against every other grouped evaluation and row update of the context, on any stream.  Its launches are not for
 * CUDA-graph capture: each cooperative launch's grid-barrier target is computed on the host.
 * b200dpf_ctx_last_device_ms times the evaluation launches only (the plan kernels, gather and scatter are outside),
 * and b200dpf_ctx_last_launches counts them.
 */
int b200dpf_group_eval_device_bins(b200dpf_ctx *ctx, const void *keys_dev, const int32_t *bins_dev, int64_t nkeys,
                                   int prf, void *out_dev, int64_t *bad_dev, void *cuda_stream);
/*
 * For tests: the lists of a grouped context's last plan.  which = 0: those b200dpf_group_eval_device_bins made on the
 * device (this waits for the context's last operation); which = 1: those the last b200dpf_group_eval or
 * b200dpf_group_eval_device made on the host.  counts receives (key groups, work units, keys, keys whose bin is out of
 * range); descs (32 bytes each: key_first, nkeys, depth, s, nsub, 0 as 32-bit words, then the bin's first row in
 * 16-byte units as 64 bits), units (4 x uint32: group, first item, items, 0) and order (2 x uint32: the caller's index
 * of the key at each sorted position, its bin's depth) receive up to their caps' entries.  ESTATE when there is no
 * such plan.
 */
int b200dpf_group_plan_lists(b200dpf_ctx *ctx, int which, int64_t *counts, void *descs, int64_t descs_cap, void *units,
                             int64_t units_cap, void *order, int64_t order_cap);
int b200dpf_group_bins(const b200dpf_ctx *ctx);

/*
 * Batch-PIR query batches: b200dpf_group_eval_device for the one shape batch PIR uses, where every query
 * carries exactly one key for every bin (dummy keys for the bins it does not need, so the server learns
 * nothing from which bins a query uses).  Works on every kind of grouped context.
 *   keys_dev: nqueries queries, query-major; query q has one key for every bin g = 0 .. nbins-1, in bin
 *             order, in one of two formats (16-byte aligned either way):
 *     B200DPF_KEYS_WIRE     int32 [nqueries][nbins][524], the format b200dpf_group_eval_device and
 *                           b200dpf_gen_batch_gpu use.
 *     B200DPF_KEYS_COMPACT  uint8 [nqueries][b200dpf_group_query_bytes(ctx)]: a query is its nbins keys back to
 *                           back, each in its kind's compact form (b200dpf_key_pack, _et or _xor) at its bin's
 *                           depth d, so b200dpf_key_packed_size(d) bytes -- always a multiple of 16.  These are
 *                           the bytes the evaluation reads: a key for a 2^10-row bin is 672 bytes of its 2096
 *                           (early-terminated: 544, XOR-shared: 224).
 *   out_dev:  int32 [nqueries][nbins][entry_size] (4-byte aligned).  out_dev[q][g] is bit for bit what
 *             b200dpf_group_eval_device (and so b200dpf_group_eval) returns for the same keys with bins =
 *             0, 1, .., nbins-1 repeated nqueries times: sums mod 2^32, or XORs on XOR-shared contexts.
 * The arguments are checked before anything is enqueued: a context that is not grouped is ESTATE; a null
 * buffer, nqueries < 1, nqueries * nbins > 2^24, an unknown prf or key_format, or a misaligned buffer is EINVAL.
 * The keys are NOT validated, as on b200dpf_group_eval_device: a key's depth comes from its bin, never from its
 * header (a compact key's magic and depth bytes are ignored too), and nothing is read beyond the key's own bytes.
 * Both buffers must stay valid until the stream reaches the end of the evaluation.
 * Ordering: the call joins the context's one-operation-in-flight chain (see "Threading" above), so it is
 * ordered against every other grouped evaluation and row update of the context, on any stream.
 * Cached plan: with one key per bin per query, the sort by bin is a fixed transpose and the whole launch plan
 * depends on nqueries alone.  It is made on the host in O(nbins + key groups + work units), kept on the device
 * in lists only this entry point uses, and reused while nqueries, prf and the context's options
 * (b200dpf_ctx_set_option, b200dpf_ctx_set_subtree_log2) stay those of its previous call.  Such a call uploads
 * nothing and never waits on the host: it only enqueues a stream wait, the key gather, the evaluation and the
 * result scatter.  A call with a new shape plans again and uploads the plan from pinned staging; before it
 * rewrites that staging it waits on the host until the previous new shape's uploads (not its kernels) have run.
 * The per-bin layout of a compact query is made and uploaded when the context is created, so no call waits for
 * it.
 * b200dpf_ctx_last_device_ms times the evaluation launches only (the gather and scatter are outside), and
 * b200dpf_ctx_last_launches counts them.
 * b200dpf_group_query_bytes: the size of one compact query; -1 on a null or non-grouped context.
 */
enum { B200DPF_KEYS_WIRE = 0, B200DPF_KEYS_COMPACT = 1 };
int64_t b200dpf_group_query_bytes(const b200dpf_ctx *ctx);
int b200dpf_group_eval_queries_device(b200dpf_ctx *ctx, const void *keys_dev, int key_format, int64_t nqueries,
                                      int prf, void *out_dev, void *cuda_stream);

/*
 * The client's side of a query batch, on the GPU: both servers' queries for b200dpf_group_eval_queries_device,
 * made from device-resident rows and seeds.  For load generators and benchmarks; works on every kind of grouped
 * context, whose kind and bin sizes shape the keys.
 *   alphas_dev: int64 [nqueries][nbins], the row of bin g that query q selects.  Any int64 is accepted: the key is
 *               the one for the low log2(n_g) bits of alphas_dev[q][g], i.e. for row alpha mod n_g.
 *   seeds_dev:  uint8 [nqueries][nbins][44], the entropy of each key (ChaCha20 key || nonce).  A real client
 *               must take them from a CSPRNG; the keys are only as secret as these bytes.
 *   out_a_dev, out_b_dev: the two servers' queries in key_format (16-byte aligned): int32 [nqueries][nbins][524]
 *               (B200DPF_KEYS_WIRE) or uint8 [nqueries][b200dpf_group_query_bytes(ctx)] (B200DPF_KEYS_COMPACT).
 * Key g of query q is bit for bit what b200dpf_gen_batch (_et, _xor: the context's kind) returns for
 * (alphas[q][g] mod n_g, n_g, seeds[q][g]), and its compact form that key's b200dpf_key_pack (_et, _xor) bytes,
 * so the outputs feed b200dpf_group_eval_queries_device unchanged.  A compact output is written only in the
 * keys' own bytes; a wire key's unused slots are written as zero.
 * The arguments are checked before anything is enqueued, in the order of b200dpf_group_eval_queries_device: a
 * context that is not grouped is ESTATE; a null buffer, nqueries < 1, nqueries * nbins > 2^24, an unknown prf or
 * key_format, or an output that is not 16-byte aligned is EINVAL.
 * Everything is enqueued on cuda_stream with no host synchronisation.  The call writes only the caller's
 * outputs: it does not join the context's one-operation-in-flight chain and leaves the cached plan of
 * b200dpf_group_eval_queries_device alone.  The per-bin query layout and the AES table it reads are made when
 * the context is created, so it never waits, on the host or on the device, for anything of the context.
 * All four buffers must stay valid until the stream reaches the end of the call.
 */
int b200dpf_group_gen_queries_device(b200dpf_ctx *ctx, const int64_t *alphas_dev, const uint8_t *seeds_dev,
                                     int64_t nqueries, int prf, int key_format, void *out_a_dev, void *out_b_dev,
                                     void *cuda_stream);

/*
 * Row updates of a live table (no counterpart in the reference, whose only way to change a row is a
 * new eval_init).  table[indices[j]] := rows[j] for j = 0 .. count-1, with NATURAL indices (the
 * numbering keys use); rows: int32 [count][entry_size].  Only the touched rows move: nothing else is
 * uploaded, re-permuted or reallocated, and every buffer and handle of the context stays valid.
 *   - Duplicates in one call: the LAST occurrence wins, on every path.
 *   - Ordering: an evaluation enqueued on the context before the update, on any stream, sees only old
 *     rows; one enqueued after it sees only new rows; none sees a mix.  The update joins the context's
 *     one-operation-in-flight chain exactly like an evaluation (see "Threading" above).
 *   - Only the entry_size live columns of a row are written; the padding of device rows stays zero.
 *   - 0 <= count < 2^31.  count == 0 is a no-op.
 *   - Scratch: the update has its own device buffer, grown on demand and kept until b200dpf_destroy
 *     (it never touches the key / result buffers or the b200dpf_host_staging memory an evaluation in
 *     flight may still read): 16 bytes per row + the temporary storage of a CUB radix sort of `count`
 *     32-bit keys, plus a copy of the list itself (12 + 4*entry_size bytes per row) on the host paths.
 *     Memory is O(count), independent of n (no n-sized claim array).
 * How each kind of context applies the list:
 *   whole table         every entry.
 *   shard (r, G)        index i is owned iff (i & (G-1)) == bitrev_g(r); every shard takes the FULL
 *                       list (as b200dpf_create takes the full table) and ignores rows it does not own;
 *                       the host path does not copy those to the GPU.
 *   b200dpf_create_multi  ENTRIES: each device applies its shard's rows; KEYS: every replica applies
 *                       every row.  All devices' copies and kernels are issued before the first
 *                       synchronisation.  Host buffers only: b200dpf_update_rows_device returns EINVAL.
 *   grouped             use b200dpf_group_update_rows; the two other entry points return ESTATE there,
 *                       and b200dpf_group_update_rows returns ESTATE on any other context.
 */

/* Host buffers, synchronous.  Every index is validated before anything is copied: EINVAL (an index
 * outside [0, n), a negative count, a null buffer) means nothing was applied. */
int b200dpf_update_rows(b200dpf_ctx *ctx, const int64_t *indices, const int32_t *rows, int64_t count);

/* Device buffers on the context's GPU, enqueued on `cuda_stream` (NULL: the default stream) with no
 * host synchronisation; the buffers must stay valid until the stream reaches the update.  Entries
 * with an index outside [0, n) are skipped (never written); the others are applied. */
int b200dpf_update_rows_device(b200dpf_ctx *ctx, const int64_t *indices_dev, const int32_t *rows_dev, int64_t count,
                               void *cuda_stream);

/* Grouped (batch-PIR) context: row indices[j] of bin bins[j] := rows[j].  Host buffers, synchronous.  A
 * bin id outside [0, nbins) or an index >= n[bin] is EINVAL, and nothing is applied.  ESTATE on a batch-code
 * context (b200dpf_batchcode_create), whose rows change in all three copies at once (b200dpf_batchcode_update_rows),
 * and on a keyword-PIR context (b200dpf_kwpir_create), whose tags must not change (b200dpf_kwpir_update). */
int b200dpf_group_update_rows(b200dpf_ctx *ctx, const int32_t *bins, const int64_t *indices, const int32_t *rows,
                              int64_t count);

/* Replaces: dpf_cpp.eval_free -> eval_free()               dpf_wrapper.cu:86-91. */
int b200dpf_destroy(b200dpf_ctx *ctx);

/*
 * Evaluate `nkeys` keys against the context's table; host buffers in and out.
 * Replaces: dpf_cpp.eval_gpu -> eval_gpu()                dpf_wrapper.cu:134-186
 *           (+ dpf_hybrid<prf>() dpf_gpu/dpf/dpf_hybrid.cu:258-272).
 * keys: int32[nkeys][524] (host).  out: int32[nkeys][entry_size] (host).
 * Synchronous: the result is complete on return.  Any nkeys >= 1 (the
 * reference requires exactly 512).
 */
int b200dpf_eval(b200dpf_ctx *ctx, const int32_t *keys, int64_t nkeys, int prf, int32_t *out);

/*
 * Same evaluation with the batch given as nkeys POINTERS to int32[524] keys -- the shape the
 * reference's eval_gpu receives (a vector of 512 key tensors, dpf_wrapper.cu:134-146).  Replaces
 * its per-key marshalling loop + blocking upload (dpf_wrapper.cu:137-150): the live parts of each
 * key are gathered into pinned staging in the compact layout and uploaded chunk by chunk while the
 * host gathers the next chunk.
 */
int b200dpf_eval_gather(b200dpf_ctx *ctx, const int32_t *const *keys, int64_t nkeys, int prf, int32_t *out);

/*
 * Same evaluation with keys in the compact wire form (b200dpf_key_pack): `packed` holds nkeys
 * keys of this table's depth back to back, b200dpf_key_packed_size(depth) bytes each (host
 * memory).  The buffer goes to the device as it is and the kernel reads the packed layout, so the
 * host-to-device copy is 2.3x smaller at n = 2^14 and 1.6x at n = 2^20 than with the
 * reference's 2096-byte keys (dpf_wrapper.cu:26-46, :150).
 */
int b200dpf_eval_packed(b200dpf_ctx *ctx, const uint8_t *packed, int64_t nkeys, int prf, int32_t *out);

/*
 * Pinned (page-locked) host staging owned by the context, sized for `nkeys` keys: callers
 * that assemble a batch from scattered keys (the reference passes 512 separate tensors,
 * dpf_wrapper.cu:137-146) can pack straight into it and hand the same pointer to
 * b200dpf_eval, which then copies to the device without an intermediate staging copy.
 * The buffer stays valid until the next b200dpf_host_staging / b200dpf_destroy.
 */
int b200dpf_host_staging(b200dpf_ctx *ctx, int64_t nkeys, int32_t **keys_pinned);

/*
 * Same computation with DEVICE buffers, enqueued on `cuda_stream` (a
 * cudaStream_t, may be NULL for the default stream) and NOT synchronised:
 * for callers that keep keys and results resident (benchmarks, NCCL reduce of
 * sharded partials).  keys_dev: int32[nkeys][524]; out_dev: int32[nkeys][entry_size].
 */
int b200dpf_eval_device(b200dpf_ctx *ctx, const void *keys_dev, int64_t nkeys, int prf,
                        void *out_dev, void *cuda_stream);

/*
 * As b200dpf_eval_device, but ADDS the results into out_dev (mod 2^32) instead
 * of overwriting it: out_dev is not cleared first.  With out_dev pointing at a
 * peer GPU's buffer (NVLink peer mapping / symmetric memory) the kernel's
 * red.global.add.u32 epilogue performs the cross-shard reduction itself, so
 * sharded evaluation needs no separate collective (SURVEY.md section 8(e),
 * "fused alternative").  The caller orders the clearing of the destination
 * before, and its consumption after, all contributing launches.  On an XOR-shared
 * context (b200dpf_create_xor) it XORs the results into out_dev instead
 * (red.global.xor.b32), the group those results live in.
 */
int b200dpf_eval_device_acc(b200dpf_ctx *ctx, const void *keys_dev, int64_t nkeys, int prf,
                            void *out_dev, void *cuda_stream);

/*
 * Non-fused full-domain expansion on the GPU (SURVEY.md section 8(f) rank 2;
 * the role of FUSES_MATMUL=0 in dpf_gpu/dpf/dpf_hybrid.cu:162-165, but in
 * natural index order): shares_dev[b][i] = low32(EvaluateFlat(key_b, i)) for
 * this context's shard rows... whole domain only (shard_count must be 1).
 * keys_dev: int32[nkeys][524]; shares_dev: int32[nkeys][n].
 */
int b200dpf_expand_device(b200dpf_ctx *ctx, const void *keys_dev, int64_t nkeys, int prf,
                          void *shares_dev, void *cuda_stream);

/* Introspection. */
int64_t b200dpf_ctx_n(const b200dpf_ctx *ctx);
int b200dpf_ctx_entry_size(const b200dpf_ctx *ctx);
int b200dpf_ctx_device(const b200dpf_ctx *ctx);

/* Device time in milliseconds of the kernels of the most recent b200dpf_eval / _eval_packed /
 * _eval_gather / _group_eval / _group_eval_device on this context (CUDA events around the launches, copies excluded);
 * negative if none. */
double b200dpf_ctx_last_device_ms(b200dpf_ctx *ctx);

/* Kernels launched by the most recent b200dpf_eval / _eval_device / _expand_device
 * call on this context (for benchmark accounting). */
int b200dpf_ctx_last_launches(const b200dpf_ctx *ctx);

/* Algorithm tuning knob, mainly for tests: log2 of the leaves one thread
 * expands depth-first per work item (0 = automatic). */
int b200dpf_ctx_set_subtree_log2(b200dpf_ctx *ctx, int s);

/*
 * Tuning knobs of a live context.  Their defaults come from the environment variables named
 * below, which are read ONCE, in b200dpf_create.
 *   "one_launch"    (B200DPF_ONE_LAUNCH, 1)     whole evaluation as one cooperative launch
 *   "frontier"      (B200DPF_FRONTIER, 1)       expand the top of the tree once per evaluation
 *   "frontier_mb"   (B200DPF_FRONTIER_MB, 256)  cap on the frontier buffer
 *   "subtree_log2"  (B200DPF_S, 0 = automatic)  as b200dpf_ctx_set_subtree_log2
 *   "lane_split"    (B200DPF_LANE_SPLIT, 1)     batches < 32 keys: lane = (key, subtree)
 *   "leaf_cache"    (B200DPF_LEAF_CACHE, 1)     entry_size > 32: expand once, MAC-only passes
 *   "leaf_cache_mb" (B200DPF_LEAF_CACHE_MB, 16384)  cap; larger batches run in chunks that fit
 *   "mac_tma"       (B200DPF_MAC_TMA, 1)        cp.async.bulk-staged MAC passes
 *   "balance_top"   (B200DPF_BALANCE_TOP, 1)    even per-block shares of the tree-top phase
 *   "top_log2"      (B200DPF_TOP_LOG2, 0 = estimate)  size of a tree-top item (log2 frontier nodes)
 *   "timing"        (B200DPF_TIMING, 0)         record per-block phase time stamps (diagnostics)
 * Results never depend on them.
 */
int b200dpf_ctx_set_option(b200dpf_ctx *ctx, const char *name, int value);

/*
 * Diagnostics ("timing" option): %globaltimer nanosecond stamps of the last single-launch
 * evaluation, 8 uint64 per block: [0] kernel start, [1] tables + clears done, [2] tree-top
 * phase done, [3] grid barrier passed, [4] main phase done, rest zero.  Synchronises the device.
 */
int b200dpf_ctx_read_timing(b200dpf_ctx *ctx, uint64_t *stamps, int max_blocks, int *nblocks);

/* ------------------------------------------------------------------------------------------- */
/* Early-terminated keys: four table rows per GGM leaf (DESIGN.md section 9).                   */
/* ------------------------------------------------------------------------------------------- */
/*
 * A leaf's 128-bit output is four 32-bit shares, one per table row, so a DPF over n rows walks a
 * tree of n/4 leaves: about a quarter of the PRF work of a standard key.  Row i is word (i & 3) of
 * leaf i >> 2.  The result is defined as for standard keys: out[b][e] = sum_i share_b[i] *
 * table[i][e] mod 2^32, so the two servers' results differ by table[alpha].
 *
 * The key is the int32[524] wire format with slot 0 = (d, 2, 0, 0) (d = log2(n) - 2 tree levels;
 * word 1 = log2 rows per leaf) and slot 130 = n.  Level-0 correction words are added lane-wise in
 * (Z/2^32)^4.  Every standard entry point refuses such a key (b200dpf_key_n / _key_depth return
 * -1, the others EINVAL), and the functions below refuse standard keys.  Evaluation uses the
 * standard entry points on a context made by b200dpf_create_et.
 */

/* Keys for row alpha of an n-row table, 8 <= n <= 2^31 a power of two.  Every draw comes from the
 * ChaCha20 DRBG of b200dpf_gen_secure; seed_len must be >= 44. */
int b200dpf_gen_et(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf,
                   int32_t *key_a, int32_t *key_b);

/* Batched b200dpf_gen_et on `nthreads` host threads (0 = one per hardware thread): seeds44 = count x
 * 44 bytes; keys_a/keys_b: int32[count][524].  Identical keys for any nthreads. */
int b200dpf_gen_batch_et(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                         int nthreads, int32_t *keys_a, int32_t *keys_b);

/* b200dpf_gen_batch_et on a GPU, with the arguments and contract of b200dpf_gen_batch_gpu: bit-identical keys
 * for the same seeds, outputs in host or device memory, n and every alpha checked before the device is opened. */
int b200dpf_gen_batch_gpu_et(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                             int device, int32_t *keys_a, int32_t *keys_b);

/* One server's share of every row on the CPU, natural order: out[i], i < n (n read from the key). */
int b200dpf_eval_cpu_et(const int32_t *key, int prf, int32_t *out_n);

/* Compact form: the layout and size (b200dpf_key_packed_size(d) = 32 + 64*d) of b200dpf_key_pack,
 * magic "DPE4".  b200dpf_key_unpack and b200dpf_eval_packed on a standard context refuse it. */
int b200dpf_key_pack_et(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written);
int b200dpf_key_unpack_et(const uint8_t *in, size_t in_len, int32_t *key);

/*
 * A context for early-terminated keys, arguments as b200dpf_create with n >= 8 and shard_count a
 * power of two <= n/8.  The device table keeps each leaf's four rows together: row 4p + l holds
 * natural row 4*bitrev(p) + l.  Shard (r, G) owns the leaves of breadth-first subtree r, i.e. row i
 * iff ((i >> 2) & (G-1)) == bitrev_g(r).  b200dpf_eval, _eval_gather, _eval_packed ("DPE4" keys),
 * _host_staging, _eval_device, _eval_device_acc, _expand_device, _update_rows, _update_rows_device,
 * _ctx_set_option and the introspection functions work on it as on a standard context (ctx_n counts
 * rows); the host paths return EINVAL for a standard key before copying anything.  The "tma_rows"
 * option has no effect here.  There is no multi-device variant; the grouped (batch-PIR) variant is
 * b200dpf_group_create_et.
 */
int b200dpf_create_et(b200dpf_ctx **ctx, const int32_t *table, int64_t n, int entry_size,
                      int device, int shard_rank, int shard_count);

/* Table rows per tree leaf: 4 on a context of b200dpf_create_et or b200dpf_group_create_et, 128 on one of
 * b200dpf_create_xor or b200dpf_group_create_xor, 1 otherwise; -1 for null. */
int b200dpf_ctx_rows_per_leaf(const b200dpf_ctx *ctx);

/* ------------------------------------------------------------------------------------------- */
/* XOR-shared keys: 128 table rows per GGM leaf (DESIGN.md section 10).                         */
/* ------------------------------------------------------------------------------------------- */
/*
 * Two-server XOR PIR (a BGI DPF with Chor et al.'s XOR reconstruction).  A leaf's 128-bit output is
 * 128 one-bit shares, one per table row, so a DPF over n rows walks a tree of n/128 leaves.  Row i is
 * bit (i & 127) of leaf i >> 7; bit b of a 128-bit value is bit (b & 31) of its little-endian word
 * b >> 5.
 *
 * THE RESULT IS AN XOR, NOT A SUM: out[b][e] = XOR over i of (share_b[i] ? table[i][e] : 0), as uint32,
 * so the two servers' results XOR to table[alpha] (out_a ^ out_b == table[alpha]).  The shares of the
 * two servers differ in exactly bit alpha.
 *
 * The key is the int32[524] wire format with slot 0 = (d, 7, 0, 0) (d = log2(n) - 7 tree levels) and
 * slot 130 = n.  Level-0 correction words are XORed in (the group (Z/2)^128).  Every standard and
 * early-terminated entry point refuses such a key, and the functions below refuse the other two kinds.
 */

/* Keys for row alpha of an n-row table, 256 <= n <= 2^31 a power of two.  Every draw comes from the
 * ChaCha20 DRBG of b200dpf_gen_secure; seed_len must be >= 44. */
int b200dpf_gen_xor(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf,
                    int32_t *key_a, int32_t *key_b);

/* Batched b200dpf_gen_xor on `nthreads` host threads (0 = one per hardware thread): seeds44 = count x
 * 44 bytes; keys_a/keys_b: int32[count][524].  Identical keys for any nthreads. */
int b200dpf_gen_batch_xor(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                          int nthreads, int32_t *keys_a, int32_t *keys_b);

/* b200dpf_gen_batch_xor on a GPU, with the arguments and contract of b200dpf_gen_batch_gpu. */
int b200dpf_gen_batch_gpu_xor(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                              int device, int32_t *keys_a, int32_t *keys_b);

/* One server's share bits of every row on the CPU, packed: bits[n / 32] in natural order, row i = bit
 * (i & 31) of bits[i >> 5] (leaf j gives words 4j .. 4j+3; n read from the key). */
int b200dpf_eval_cpu_xor(const int32_t *key, int prf, uint32_t *bits);

/* Compact form: the layout and size (b200dpf_key_packed_size(d) = 32 + 64*d) of b200dpf_key_pack,
 * magic "DPX7".  The standard and early-terminated unpack and packed-evaluation paths refuse it. */
int b200dpf_key_pack_xor(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written);
int b200dpf_key_unpack_xor(const uint8_t *in, size_t in_len, int32_t *key);

/*
 * A context for XOR-shared keys, arguments as b200dpf_create with n >= 256 and shard_count a power of
 * two <= n/256.  The device table keeps each leaf's 128 rows together: row 128p + l holds natural row
 * 128*bitrev(p) + l.  Shard (r, G) owns row i iff ((i >> 7) & (G-1)) == bitrev_g(r); the shards' results
 * XOR to the whole table's.  On it:
 *   b200dpf_eval, _eval_gather, _eval_packed ("DPX7" keys), _host_staging, _eval_device, _update_rows,
 *   _update_rows_device, _ctx_set_option and the introspection functions work as on an early-terminated
 *   context, with the XOR result above; the host paths return EINVAL for a key of another kind before
 *   copying anything;
 *   b200dpf_eval_device_acc XORs the results into out_dev (red.global.xor) instead of adding them;
 *   b200dpf_expand_device writes the packed share bits, shares_dev = uint32[nkeys][n / 32] as
 *   b200dpf_eval_cpu_xor.
 * Entries are evaluated 16 columns per pass; wider entries take one pass (one tree walk) per 16 columns,
 * so the "leaf_cache", "leaf_cache_mb", "mac_tma" and "tma_rows" options have no effect here.  The
 * grouped (batch-PIR) variant is b200dpf_group_create_xor; there is no multi-device or GPU-keygen
 * variant.
 */
int b200dpf_create_xor(b200dpf_ctx **ctx, const int32_t *table, int64_t n, int entry_size,
                       int device, int shard_rank, int shard_count);

/* ------------------------------------------------------------------------------------------- */
/* Trimmed tables: any row count, no padding to a power of two (DESIGN.md section 11).          */
/* ------------------------------------------------------------------------------------------- */
/*
 * The contexts above need a power-of-two row count; padding a table with zero rows up to one costs as
 * much device memory and evaluation work as real rows.  A trimmed context takes a table of any n rows,
 * 1 <= n <= 2^31, for keys of any kind, and numbers rows so that the live rows come first in the tree:
 * row r sits at leaf position r >> b (b = log2 rows per leaf: 0 standard, 2 early-terminated, 7
 * XOR-shared), so the work past the last live row is never issued.  The client reaches row r with an
 * ordinary key of the kind (b200dpf_gen_secure, _gen_et, _gen_xor and their batched and GPU forms), made
 * for n = b200dpf_trimmed_domain(n) rows and alpha = b200dpf_trimmed_alpha(r, n, kind); keygen, the key
 * formats and packing are unchanged.  The result is then, with share_b the key's CPU share vector over
 * the domain (b200dpf_eval_cpu, _et, _xor):
 *   out[b][e] = sum over r < n of share_b[trimmed_alpha(r)] * table[r][e]  mod 2^32   (XOR-shared: XOR)
 * so the two servers' results reconstruct table[r] for the key of row r.
 *
 * Padding bound: the device table holds b200dpf_ctx_table_rows = n rounded up to a multiple of 2^g rows
 * (per bin on a grouped context), with N = b200dpf_trimmed_domain(n) and
 *   g = min(log2 N, max(log2 N - 7, b + m)),   m = 6 for standard and early-terminated keys, 1 for XOR-shared,
 * so the padding is below max(N / 128, 2^(b + m)) rows: under n / 64 (1.6 %) once n > 2^(b + m + 7), and at
 * most 63 rows (standard), 255 (early-terminated) or 255 (XOR-shared) on a bin that small.  Work items are
 * sized so that none reaches past those rows.
 */
enum { B200DPF_KIND_STANDARD = 0, B200DPF_KIND_ET = 1, B200DPF_KIND_XOR = 2 };

/* The key domain of a trimmed n-row table: the next power of two >= n, at least the kind's smallest key
 * (2 standard, 8 early-terminated, 256 XOR-shared).  -1 for n outside [1, 2^31] or an unknown kind. */
int64_t b200dpf_trimmed_domain(int64_t n, int kind);

/* The key index of row `row` of a trimmed n-row table: bitrev_d(row >> b) << b | (row & (2^b - 1)), with
 * d = log2(b200dpf_trimmed_domain(n, kind)) - b.  -1 for n outside [1, 2^31], an unknown kind or a row
 * outside [0, n).  Distinct rows have distinct indices in [0, trimmed_domain). */
int64_t b200dpf_trimmed_alpha(int64_t row, int64_t n, int kind);

/*
 * A trimmed context of `kind` (B200DPF_KIND_*) on device `device`.  table: int32 [n][entry_size] in row
 * order, host or device memory, 1 <= n <= 2^31, entry_size as b200dpf_create.  On it b200dpf_eval,
 * _eval_gather, _eval_packed (the kind's compact keys), _host_staging, _eval_device, _eval_device_acc, the
 * option setters, timing and introspection work as on a context of the kind, taking only keys of the kind
 * for n = b200dpf_trimmed_domain(n) rows (any other key is EINVAL on the host paths, before anything is
 * copied).  b200dpf_update_rows and _update_rows_device take ROW numbers r: the host path is EINVAL for
 * r outside [0, n), the device path skips such entries.  b200dpf_ctx_n is n.  b200dpf_expand_device is
 * ESTATE.  There is no sharded or multi-device trimmed context.
 */
int b200dpf_create_trimmed(b200dpf_ctx **ctx, const int32_t *table, int64_t n, int entry_size, int device,
                           int kind);

/*
 * A trimmed grouped (batch-PIR) context: bins of any size n[g] in [1, 2^31], each numbered as above.
 * b200dpf_group_eval, _group_eval_device, _group_eval_queries_device (both formats), _group_query_bytes and
 * _group_update_rows (row numbers, EINVAL for r >= n[g]) work as on a grouped context of the kind; the key
 * of bin g is for b200dpf_trimmed_domain(n[g]) rows.  b200dpf_group_gen_queries_device makes key (q, g)
 * for row alphas[q][g] mod n[g] (a non-negative modulo), i.e. the key b200dpf_gen_batch_secure (_et, _xor)
 * returns for (b200dpf_trimmed_alpha(row, n[g], kind), b200dpf_trimmed_domain(n[g], kind)); its compact
 * form is that key's b200dpf_key_pack (_et, _xor) bytes.
 */
int b200dpf_group_create_trimmed(b200dpf_ctx **ctx, const int32_t *const *tables, const int64_t *n, int nbins,
                                 int entry_size, int device, int kind);

/* 1 on a trimmed context, 0 on any other, -1 for null. */
int b200dpf_ctx_trimmed(const b200dpf_ctx *ctx);

/* ------------------------------------------------------------------------------------------- */
/* Batch codes: any k rows of one table per query (DESIGN.md section 13).                       */
/* ------------------------------------------------------------------------------------------- */
/*
 * A probabilistic batch code (Angel et al., "PIR with compressed queries and amortized query processing", 2018): the
 * server stores every row of an n-row table in 3 of nbins bins; a client that wants k rows assigns them to distinct
 * bins (a bipartite matching) and sends one key per bin.  With nbins about 1.5 k every row is placed with high
 * probability, and the server's work is 3n rows per query instead of k n for k separate queries.
 *
 * Layout.  Parameters: n rows (1 <= n <= 2^31), nbins = B (1 <= B <= min(n, 2^20)) and a public 64-bit layout_seed.
 *   mix(z)       the SplitMix64 finalizer on 64-bit words: z ^= z >> 30; z *= 0xbf58476d1ce4e5b9; z ^= z >> 27;
 *                z *= 0x94d049bb133111eb; z ^= z >> 31.
 *   h            the smallest h >= 1 with 2^(2h) >= n (so 2h >= max(2, ceil(log2 n))).
 *   F_c(x)       copy c's balanced Feistel network over 2h bits: L = x >> h, R = x mod 2^h; for rounds i = 0, 1, 2, 3:
 *                (L, R) := (R, L ^ (mix(layout_seed ^ mix(((c * 8 + i) << 32) | R)) mod 2^h)); then x = (L << h) | R.
 *   pi_c(r)      x = F_c(r), repeated (x = F_c(x)) until x < n: cycle walking makes pi_c a permutation of [0, n).
 *   m_j          ceil((n - j) / B), the x in [0, n) with x mod B = j.
 *   copy c of r  (c = 0, 1, 2) with x = pi_c(r): bin j = x mod B, row c * m_j + floor(x / B) of that bin.
 * Bin j holds exactly 3 m_j rows, every one a copy of a table row; 3 m_0 (the largest) must be <= 2^31.  The bins are
 * those of a trimmed grouped context (b200dpf_group_create_trimmed), so a client reaches row t of bin j with the key of
 * its kind for (b200dpf_trimmed_alpha(t, 3 m_j, kind), b200dpf_trimmed_domain(3 m_j, kind)).  A client locates a row's
 * copies from (n, B, layout_seed) alone.
 *
 * Privacy.  Every query carries exactly one key for every bin, whichever rows it wants; a bin no wanted row uses gets a
 * key for its row 0, which its key hides like any other row.  The layout and its seed are public and depend on no
 * query.  The plan -- which wanted row went to which bin, and which rows could not be placed -- stays with the client:
 * the server sees keys only.
 */

/* A batch-code context of `kind` (B200DPF_KIND_*) on `device`: a trimmed grouped context with the nbins bins of the
 * layout above, of 3 m_j rows each.  table: int32 [n][entry_size], host or device memory; entry_size as b200dpf_create.
 * The bins are written into the context's device table by a scatter kernel, one table row to its three copies; a host
 * table goes up in chunks of at most 64 MiB, and no other copy of the replicated table is made.  b200dpf_group_eval,
 * _group_eval_device, _group_eval_device_bins, _group_eval_queries_device, _group_gen_queries_device, _group_query_bytes,
 * the option setters, timing and introspection work on it as on any trimmed grouped context of the kind.
 * b200dpf_group_update_rows returns ESTATE on it (one copy of a row cannot change alone): use
 * b200dpf_batchcode_update_rows.  EINVAL for n, nbins or a bin size out of range, as above. */
int b200dpf_batchcode_create(b200dpf_ctx **ctx, const int32_t *table, int64_t n, int entry_size, int nbins,
                             uint64_t layout_seed, int device, int kind);

/* The public parameters of a batch-code context, which a client needs: n, nbins and layout_seed.  ESTATE on any other
 * context. */
int b200dpf_batchcode_layout(const b200dpf_ctx *ctx, int64_t *n, int *nbins, uint64_t *layout_seed);

/* Host only, no context: bins3[c] and rows3[c] receive the bin and the in-bin row of copy c = 0, 1, 2 of `row`.  EINVAL
 * for a layout out of range or a row outside [0, n). */
int b200dpf_batchcode_locate(int64_t n, int nbins, uint64_t layout_seed, int64_t row, int32_t *bins3, int64_t *rows3);

/*
 * The client's plan of nqueries queries of k wanted rows each, in host memory.
 *   wanted: int64 [nqueries][k], rows in [0, n) (any other is EINVAL before anything is written).
 *   alphas: int64 [nqueries][nbins] receives the in-bin row to query in each bin (0 in a bin no wanted row uses).
 *   slots:  int32 [nqueries][k] receives the bin whose answer is wanted row i, or -1 when it could not be placed.
 * Per query, a maximum matching of the wanted rows to distinct bins: Kuhn's augmenting paths, started from the wanted
 * rows in order, a search from row u trying its copies 0, 1, 2 in order (depth first, each bin visited at most once
 * per search, a taken bin tried by moving its row along its own copies).  A row that repeats an earlier wanted row of
 * the same query shares that row's slot (and is -1 with it).  Deterministic: the same arguments give the same bytes.
 * Limits: 1 <= k <= 4096, 1 <= nqueries, nqueries * nbins <= 2^24; the layout as for b200dpf_batchcode_create.
 */
int b200dpf_batchcode_plan(int64_t n, int nbins, uint64_t layout_seed, const int64_t *wanted, int64_t nqueries, int k,
                           int64_t *alphas, int32_t *slots);

/* The same plan on the context's GPU for load generators, one thread per query, in device buffers (wanted_dev and
 * alphas_dev 8-byte aligned, slots_dev 4-byte aligned): alphas_dev and slots_dev are bit for bit what
 * b200dpf_batchcode_plan writes, except that a wanted row outside [0, n) gets slot -1 instead of failing the call.  The
 * matching is built in alphas_dev and slots_dev themselves, so no scratch grows with nqueries.  alphas_dev feeds
 * b200dpf_group_gen_queries_device unchanged.  Enqueued on cuda_stream with no host wait; it writes only the caller's
 * buffers and, like b200dpf_group_gen_queries_device, does not join the context's one-operation-in-flight chain.
 * ESTATE on a context that is not a batch code; EINVAL for the limits of b200dpf_batchcode_plan, a null or misaligned
 * buffer. */
int b200dpf_batchcode_plan_device(b200dpf_ctx *ctx, const int64_t *wanted_dev, int64_t nqueries, int k, int64_t *alphas_dev,
                                  int32_t *slots_dev, void *cuda_stream);

/* Row updates of a batch-code context: table row indices[j] := rows[j] in all three copies, the last occurrence of a row
 * winning.  Host buffers, synchronous, ordered against evaluations as b200dpf_group_update_rows is (it takes the same
 * path, three entries per row).  An index outside [0, n), a negative count or more than (2^31 - 1) / 3 rows is EINVAL
 * before anything is applied; ESTATE on any other context. */
int b200dpf_batchcode_update_rows(b200dpf_ctx *ctx, const int64_t *indices, const int32_t *rows, int64_t count);

/* ------------------------------------------------------------------------------------------- */
/* Keyword PIR: a value by its 64-bit keyword in one query (DESIGN.md section 14).              */
/* ------------------------------------------------------------------------------------------- */
/*
 * A cuckoo hash table of n (keyword, value) items in three tables of m slots: the server places each item in one of
 * its keyword's three candidate slots; a client computes the three slots from public parameters, sends one key per
 * table, and keeps the answer whose stored keyword matches.  The server evaluates 3m rows per query.
 *
 * Layout.  Parameters: n items (1 <= n <= 2^30), m slots per table (ceil(n / 3) <= m <= 2^31), a public 64-bit
 * layout_seed and E value columns (1 <= E <= 4094).  All arithmetic is mod 2^64.
 *   mix(z)       the SplitMix64 finalizer of the batch-code layout above.
 *   h_c(w)       for c = 0, 1, 2: ((mix(mix(w ^ layout_seed) ^ ((c + 1) * 0x9E3779B97F4A7C15)) >> 32) * m) >> 32, a row
 *                in [0, m) (the product is below 2^63 because m <= 2^31).
 *   context      a trimmed grouped context (b200dpf_group_create_trimmed) of 3 bins of m rows, entry size E + 2.
 *   row format   item (w, value) sits in bin c at row h_c(w) for one c: columns [0, E) are value, column E the low and
 *                column E + 1 the high 32 bits of the tag w + 1.  An empty slot is all zeros, so tag 0 means empty
 *                and keyword 2^64 - 1 is refused.  The tag is the whole keyword: "found" is exact.
 * Keywords wider than 64 bits must be hashed down by the caller; two that hash to the same 64 bits are one keyword.
 * E = 14 keeps the context at 16 columns, the best-shaped evaluation; E = 16 makes 18 columns, which take the wide-entry
 * path.
 *
 * Placement.  A pure function of the keywords in caller order, m and layout_seed: item i is its position in the
 * caller's arrays; choice[i] in {0, 1, 2} starts at 0 and every item starts homeless.  Each round, every homeless item
 * i bids for slot (choice[i], h_choice[i](w_i)); each slot bid on goes to its smallest bidding index, whose bid takes
 * it; the slot's previous owner, if any, and every losing bidder advance choice by 1 mod 3 and are homeless in the next
 * round.  The placement ends when no item is homeless.  A round's outcome depends only on the set of homeless items,
 * so it does not depend on thread scheduling, device or stream.  After 1024 rounds with items still homeless the
 * create fails with B200DPF_EFULL and creates nothing; another layout_seed or a larger m is the remedy (the Python
 * layer retries layout_seed + 1, + 2, ..., 8 seeds in all).  DESIGN.md section 14 gives the rounds a build takes;
 * m = ceil(1.3 n / 3), the Python default, stays far below the cap.
 *
 * Privacy.  Every query carries exactly one key for each of the three bins, whether or not its keyword is present.
 * The layout and its seed are public and depend on no query.  The client learns the full rows of its three candidate
 * slots, which may hold other keywords' items; like index PIR, this does not hide the database from the client.
 */

/* A keyword-PIR context of `kind` (B200DPF_KIND_*) on `device`, laid out as above.  keywords: uint64 [n], values: int32
 * [n][value_size], each in host or device memory; keywords and values on the context's device are read in place, host
 * values go up in chunks of at most 64 MiB.  Duplicate keywords and keyword 2^64 - 1 are EINVAL (found by a radix
 * sort on the device, before placement).  The placement runs on the GPU, one bid and one resolve kernel per round;
 * its O(n + m) scratch is freed before the call returns.  Synchronous.  B200DPF_EFULL when the placement does not
 * finish (above).  b200dpf_group_eval, _group_eval_device, _group_eval_device_bins, _group_eval_queries_device,
 * _group_gen_queries_device, _group_query_bytes, the option setters, timing and introspection work on it as on any
 * trimmed grouped context of the kind; b200dpf_group_update_rows returns ESTATE on it (use b200dpf_kwpir_update). */
int b200dpf_kwpir_create(b200dpf_ctx **ctx, const uint64_t *keywords, const int32_t *values, int64_t n, int value_size, int64_t m,
                         uint64_t layout_seed, int device, int kind);

/* The public parameters of a keyword-PIR context, which a client needs: n, m, layout_seed and value_size (E).  ESTATE
 * on any other context. */
int b200dpf_kwpir_layout(const b200dpf_ctx *ctx, int64_t *n, int64_t *m, uint64_t *layout_seed, int *value_size);

/* The rounds the context's placement took, and their time on the device by CUDA events (the per-round host reads of
 * the homeless count included, the duplicate check and the row scatter not).  ESTATE on any other context. */
int b200dpf_kwpir_build_stats(const b200dpf_ctx *ctx, int *rounds, double *place_ms);

/* Host only, no context: rows3[j][c] = h_c(keywords[j]), the in-bin row to query in bin c, for count keywords.
 * EINVAL for m outside [1, 2^31], a negative count, a null buffer or keyword 2^64 - 1. */
int b200dpf_kwpir_locate(int64_t m, uint64_t layout_seed, const uint64_t *keywords, int64_t count, int64_t *rows3);

/* The same rows on the context's GPU for load generators, one thread per query: keywords_dev uint64 [nqueries] into
 * alphas_dev int64 [nqueries][3] (both 8-byte aligned), which feeds b200dpf_group_gen_queries_device unchanged.
 * Keyword 2^64 - 1 gets its rows like any other (it is never found).  Enqueued on cuda_stream with no host wait; it
 * writes only the caller's buffers and does not join the context's one-operation-in-flight chain.  ESTATE on any other
 * context; EINVAL for a null or misaligned buffer or nqueries outside [1, 2^24 / 3]. */
int b200dpf_kwpir_plan_device(b200dpf_ctx *ctx, const uint64_t *keywords_dev, int64_t nqueries, int64_t *alphas_dev,
                              void *cuda_stream);

/* Value updates of a keyword-PIR context: the value of keywords[j] := values[j] (int32 [count][value_size]), the last
 * occurrence of a keyword winning.  Host buffers, synchronous.  A kernel finds each keyword's slot from the tags of its
 * three candidate rows; a keyword that is not in the table (or 2^64 - 1), a negative count or one of 2^31 or more is
 * EINVAL before anything is applied.  The rows then take the path of b200dpf_group_update_rows, ordered against
 * evaluations as it is.  Keywords cannot be inserted or deleted: that needs a new context.  ESTATE on any other
 * context. */
int b200dpf_kwpir_update(b200dpf_ctx *ctx, const uint64_t *keywords, const int32_t *values, int64_t count);

/* Introspection: tags[c][r] (uint64 [3][m], host memory) receives the tag stored in row r of bin c, w + 1 for the item
 * of keyword w placed there or 0 for an empty slot.  Synchronous.  ESTATE on any other context. */
int b200dpf_kwpir_tags(const b200dpf_ctx *ctx, uint64_t *tags);

/* Rows of the context's device table, padding included (on a grouped context all bins together; on a
 * multi-device context one device's); -1 for null.  A context that is not trimmed pads nothing: n (a
 * shard: n / shard_count). */
int64_t b200dpf_ctx_table_rows(const b200dpf_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* B200DPF_H */
