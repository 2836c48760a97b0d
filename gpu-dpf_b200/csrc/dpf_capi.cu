/*
 * dpf_capi.cu -- implementation of the C ABI declared in include/b200dpf.h.
 *
 * Owns the device state of one table (or one entry-range shard of it) and
 * turns b200dpf_eval* calls into launches of the sm_90a kernel in
 * dpf_kernels.cu.  The GPU entry points have no CPU fallback: without a usable
 * CUDA device they fail with B200DPF_ECUDA.
 */
#include "b200dpf.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <new>
#include <optional>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "dpf_host.h"
#include "dpf_kernels.cuh"

using namespace b200dpf;

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return code;
}

#define CUDA_TRY(expr)                                                                        \
    do {                                                                                      \
        cudaError_t e__ = (expr);                                                             \
        if (e__ != cudaSuccess)                                                               \
            return fail(B200DPF_ECUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e__),       \
                        __FILE__, __LINE__);                                                  \
    } while (0)

int ilog2(int64_t v)
{
    int b = 0;
    while (((int64_t)1 << b) < v) b++;
    return b;
}

uint32_t bitrev_host(uint32_t v, int bits)
{
    uint32_t r = 0;
    for (int i = 0; i < bits; i++) r |= ((v >> i) & 1u) << (bits - 1 - i);
    return r;
}

struct DeviceGuard {
    int prev = -1;
    bool ok = false;
    explicit DeviceGuard(int dev)
    {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        ok = cudaSetDevice(dev) == cudaSuccess;
    }
    ~DeviceGuard()
    {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

/* A grow-only allocation of device memory (cudaMalloc) or, if Pinned, page-locked host memory
 * (cudaMallocHost), freed by its destructor. */
template <class T, bool Pinned>
struct Buffer {
    T *ptr = nullptr;
    size_t cap = 0;   /* bytes */
    Buffer() = default;
    Buffer(Buffer &&o) noexcept : ptr(std::exchange(o.ptr, nullptr)), cap(std::exchange(o.cap, 0)) {}
    ~Buffer() { release(); }
    void release()
    {
        if (ptr && Pinned) cudaFreeHost(ptr);
        else if (ptr) cudaFree(ptr);
        ptr = nullptr;
        cap = 0;
    }
    /* at least `bytes`; a smaller buffer is replaced (its contents are lost) and *grown says so */
    int reserve(size_t bytes, bool *grown = nullptr)
    {
        if (grown) *grown = false;
        if (bytes <= cap) return B200DPF_OK;
        release();
        if (Pinned) CUDA_TRY(cudaMallocHost(&ptr, bytes));
        else CUDA_TRY(cudaMalloc(&ptr, bytes));
        cap = bytes;
        if (grown) *grown = true;
        return B200DPF_OK;
    }
};
template <class T> using DeviceBuffer = Buffer<T, false>;
template <class T> using PinnedBuffer = Buffer<T, true>;

constexpr size_t kKeyBytes = host::KEY_WORDS * sizeof(int32_t);   /* one key in the wire format */

}  // namespace

struct SmemLayoutCache;   /* per (prf, nv, mode) launch layouts, filled on first use */
struct MultiState;        /* b200dpf_create_multi: per-device sub-contexts + worker threads */

struct GroupBins {            /* b200dpf_group_create: many tables ("bins") behind one context */
    std::vector<int64_t> n;
    std::vector<int> depth;
    std::vector<uint64_t> row_off;     /* first row of the bin in d_table */
    DeviceBuffer<GroupDesc> d_descs;   /* both hold at least 1,024 descriptors */
    PinnedBuffer<GroupDesc> h_descs;
    std::vector<int64_t> perm;         /* sorted position -> caller's index, of the last evaluation */
    DeviceBuffer<uint2> d_bin_info;    /* [nbins] (row_off, depth) for row updates, uploaded on first use */
};

struct b200dpf_ctx {
    std::unique_ptr<MultiState> multi;   /* non-null: this context only fans out to multi->sub[] */
    std::unique_ptr<GroupBins> bins;     /* non-null: grouped (batch-PIR) context, use b200dpf_group_eval */
    std::unique_ptr<SmemLayoutCache> layouts;
    int device = 0;
    int64_t n = 0;
    int depth = 0;
    int entry_size = 0;
    int entry_pad = 0;       /* row length in int32: 16, 32 or a multiple of 64     */
    int shard_rank = 0, shard_count = 1, shard_bits = 0;
    int64_t n_local = 0;
    int depth_local = 0;
    /* log2 table rows per tree leaf: 0, or 2 on an early-terminated context (b200dpf_create_et).  n,
     * n_local, the table, the leaf cache and the results count rows; depth, depth_local, the shards,
     * the work items and the frontier count leaves. */
    int lane_bits = 0;
    DeviceBuffer<int32_t> d_table;
    cudaStream_t stream = nullptr;
    DeviceBuffer<int32_t> d_keys;     /* whole wire-format keys */
    DeviceBuffer<int32_t> d_out;
    DeviceBuffer<uint32_t> d_counters;
    DeviceBuffer<void> d_frontier;
    DeviceBuffer<uint32_t> d_leaf_cache;
    PinnedBuffer<int32_t> h_keys;     /* staging: whole wire-format keys, at least 512 */
    PinnedBuffer<int32_t> h_out;      /* staging: at least 8,192 int32 */
    int sm_count = 0;
    uint32_t smem_base = 0;
    int last_launches = 0;
    /* tuning knobs: defaults from the environment, read ONCE at b200dpf_create; changed per
     * context with b200dpf_ctx_set_option */
    struct Knobs {
        int leaf_cache = 1;        /* B200DPF_LEAF_CACHE     wide entries: cache leaves, MAC-only passes  */
        int leaf_cache_mb = 16384; /* B200DPF_LEAF_CACHE_MB  cap; larger batches are evaluated in chunks   */
        int lane_split = 1;        /* B200DPF_LANE_SPLIT     batches < 32 keys: lane = (key, subtree)      */
        int frontier = 1;          /* B200DPF_FRONTIER       expand the tree top once per evaluation       */
        int frontier_mb = 256;     /* B200DPF_FRONTIER_MB                                                  */
        int subtree_log2 = 0;      /* B200DPF_S              0 = automatic                                  */
        int mac_tma = 1;           /* B200DPF_MAC_TMA        cp.async.bulk-staged MAC passes               */
        int one_launch = 1;        /* B200DPF_ONE_LAUNCH     whole evaluation as one cooperative launch    */
        int balance_top = 1;       /* B200DPF_BALANCE_TOP    even per-block shares of the tree-top phase    */
        int timing = 0;            /* B200DPF_TIMING         per-block phase time stamps (diagnostics)      */
        int top_log2 = 0;          /* B200DPF_TOP_LOG2       log2 leaves-of-the-frontier per tree-top item (0 = estimate) */
        int tma_rows = 0;          /* B200DPF_TMA_ROWS       fused kernel: stage each item's rows with cp.async.bulk
                                                             (16-column tables, Salsa/ChaCha/dummy); on an H100 at n=2^20
                                                             +4 % for Salsa20, -2 % for ChaCha20 against broadcast
                                                             loads, other sizes unmeasured -- so off */
    } knobs;
    DeviceBuffer<unsigned long long> d_timing;   /* [blocks][8] */
    int coop_ok = 0;               /* device supports cooperative launches                                 */
    DeviceBuffer<uint32_t> d_top_counters;  /* top-phase tickets: zero between launches (self re-arming)   */
    DeviceBuffer<uint32_t> d_gridbar;       /* monotonic arrival counter of the in-kernel grid barrier      */
    uint32_t bar_epoch = 0;               /* value d_gridbar holds when no launch is in flight              */
    bool coop_state_dirty = true;         /* top tickets / barrier counter must be cleared before use       */
    /* one evaluation in flight per context: launches on a different stream than the previous
     * evaluation first wait for it (the scratch buffers above are shared)                                 */
    cudaEvent_t ev_done = nullptr;
    cudaStream_t last_stream = nullptr;
    bool has_last = false;
    /* device time of the last host-buffer evaluation (first launch .. last launch), for callers that
     * want the kernel time next to their own wall clock */
    cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;
    bool timed = false;
    /* row updates (b200dpf_update_rows*): their own scratch, so an update never touches a buffer an
     * evaluation in flight may read; layout at UpdateLayout */
    DeviceBuffer<char> d_update;
    ~b200dpf_ctx();   /* the members free the buffers; this destroys the stream and events */
};

namespace {

struct SmemLayout {
    int threads, blocks_per_sm, grid;
    int budget;               /* dynamic shared memory one block may use */
    size_t smem_fixed;        /* AES: whole budget; others: computed from s */
    uint32_t off_meta;        /* correction words, meta_cw bytes                          */
    uint32_t off_small;       /* level-0 low words, root seeds and flag (kMetaSmall bytes) */
    uint32_t off_lo, off_hi, off_tab, meta_cw, level_bytes;
    int cap_lo, cap_hi, s_max;
};

}  // namespace

struct SmemLayoutCache {
    SmemLayout entry[4][3][MODE_COUNT];
    bool valid[4][3][MODE_COUNT] = {};
};

namespace {

int smem_layout_compute(b200dpf_ctx *c, int prf, int nv, int mode, SmemLayout *L);

/* Dynamic shared memory layout of the kernel instantiated for (prf, nv, mode); the CUDA
 * attribute queries behind it are made once per context. */
int smem_layout(b200dpf_ctx *c, int prf, int nv, int mode, SmemLayout *L)
{
    const int ni = nv == 4 ? 0 : (nv == 8 ? 1 : 2);
    if (!c->layouts) c->layouts.reset(new (std::nothrow) SmemLayoutCache());
    if (c->layouts && c->layouts->valid[prf][ni][mode]) {
        *L = c->layouts->entry[prf][ni][mode];
        return B200DPF_OK;
    }
    const int rc = smem_layout_compute(c, prf, nv, mode, L);
    if (rc == B200DPF_OK && c->layouts) {
        c->layouts->entry[prf][ni][mode] = *L;
        c->layouts->valid[prf][ni][mode] = true;
    }
    return rc;
}

int smem_layout_compute(b200dpf_ctx *c, int prf, int nv, int mode, SmemLayout *L)
{
    std::memset(L, 0, sizeof *L);
    L->threads = eval_threads(prf, nv);
    L->blocks_per_sm = eval_min_blocks(prf, nv);
    L->grid = c->sm_count * L->blocks_per_sm;
    int max_smem = 0;
    CUDA_TRY(eval_max_smem(prf, nv, mode, &max_smem));
    int sm_total = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&sm_total, cudaDevAttrMaxSharedMemoryPerMultiprocessor, c->device));
    /* every resident block also pays the 1 KiB system reservation */
    int budget = std::min(max_smem, sm_total / L->blocks_per_sm - 1024);
    budget &= ~15;
    L->budget = budget;

    L->meta_cw = (uint32_t)c->depth * 4u * 32u * 16u;
    const uint32_t kMetaSmall = 512u + 512u + 16u;
    const uint32_t meta = L->meta_cw + kMetaSmall;
    L->level_bytes = (uint32_t)L->threads * 16u;
    if (prf == B200DPF_PRF_AES128) {
        /* tables: 128 KiB whose shared-window address is 64 KiB aligned */
        const uint32_t tab_abs = (c->smem_base + 65535u) & ~65535u;
        const uint32_t off_tab = tab_abs - c->smem_base;
        const uint32_t a_size = off_tab;                         /* region A: before the tables */
        const uint32_t b_off = off_tab + 131072u;                /* region B: after them        */
        if ((int64_t)budget < (int64_t)b_off) return fail(B200DPF_ECUDA, "shared memory too small for AES tables");
        const uint32_t b_size = (uint32_t)budget - b_off;
        L->off_tab = off_tab;
        uint32_t a_used = 0, b_used = 0;
        if (meta <= a_size) { L->off_meta = 0; L->off_small = L->meta_cw; a_used = meta; }
        else if (meta <= b_size) { L->off_meta = b_off; L->off_small = b_off + L->meta_cw; b_used = meta; }
        else if (L->meta_cw <= a_size && kMetaSmall <= b_size) {
            /* depth 31: the correction words alone fill region A, so the rest goes after the tables */
            L->off_meta = 0; a_used = L->meta_cw;
            L->off_small = b_off; b_used = kMetaSmall;
        }
        else return fail(B200DPF_EINVAL, "depth %d needs more shared memory than available", c->depth);
        a_used = (a_used + 15u) & ~15u;
        b_used = (b_used + 15u) & ~15u;
        L->off_lo = b_off + b_used;
        L->cap_lo = (int)((b_size - b_used) / L->level_bytes);
        L->off_hi = a_used;
        L->cap_hi = (int)((a_size - a_used) / L->level_bytes);
        L->smem_fixed = (size_t)budget;
    } else {
        L->off_meta = 0;
        L->off_small = L->meta_cw;
        L->off_lo = (meta + 15u) & ~15u;
        if ((int64_t)budget < (int64_t)L->off_lo) return fail(B200DPF_EINVAL, "depth %d needs more shared memory than available", c->depth);
        L->cap_lo = (int)(((uint32_t)budget - L->off_lo) / L->level_bytes);
        L->off_hi = L->off_lo;
        L->cap_hi = 0;
        L->smem_fixed = 0;
    }
    L->s_max = 1 + L->cap_lo + L->cap_hi;
    return B200DPF_OK;
}

/* s = the deepest pending-sibling stack any phase of the launch needs */
void fill_common(const b200dpf_ctx *c, const SmemLayout &L, int s, int64_t nkeys, int kpw_log2, EvalParams *p,
                 size_t *smem)
{
    std::memset(p, 0, sizeof *p);
    p->depth = c->depth;
    p->nkeys = (int)nkeys;
    p->kpw_log2 = kpw_log2;
    p->key_groups = (int)((nkeys + (1 << kpw_log2) - 1) >> kpw_log2);
    p->table = reinterpret_cast<const uint4 *>(c->d_table.ptr);
    p->row_stride_v = (uint32_t)c->entry_pad / 4u;
    p->out_stride = (uint32_t)c->entry_size;
    p->n = (uint64_t)c->n;
    p->off_cw = L.off_meta;
    p->off_cwlo = L.off_small;
    p->off_root = p->off_cwlo + 512u;
    p->off_flag = p->off_root + 512u;
    p->off_stack_lo = L.off_lo;
    p->off_stack_hi = L.off_hi;
    p->off_tab = L.off_tab;
    *smem = L.smem_fixed ? L.smem_fixed : (size_t)L.off_lo + (size_t)(s > 1 ? s - 1 : 0) * L.level_bytes;
}

int env_int(const char *name, int dflt)
{
    const char *v = std::getenv(name);
    return (v && *v) ? std::atoi(v) : dflt;
}

/* One operation in flight per context: its scratch buffers are shared.  Work about to be enqueued on
 * `stream` first waits for the context's last operation when that ran on another stream. */
int wait_last(b200dpf_ctx *c, cudaStream_t stream)
{
    if (c->has_last && c->last_stream != stream) CUDA_TRY(cudaStreamWaitEvent(stream, c->ev_done, 0));
    return B200DPF_OK;
}

/* The work enqueued on `stream` so far becomes the context's last operation. */
int mark_last(b200dpf_ctx *c, cudaStream_t stream)
{
    CUDA_TRY(cudaEventRecord(c->ev_done, stream));
    c->last_stream = stream;
    c->has_last = true;
    return B200DPF_OK;
}

/* Pinned staging never shrinks below 512 keys or 8,192 result elements. */
int reserve_host_keys(b200dpf_ctx *c, size_t key_bytes)
{
    return c->h_keys.reserve(std::max<size_t>((key_bytes + kKeyBytes - 1) / kKeyBytes, 512) * kKeyBytes);
}

int reserve_host_out(b200dpf_ctx *c, size_t out_elems)
{
    return c->h_out.reserve(std::max<size_t>(out_elems, 8192) * sizeof(int32_t));
}

/* device key / result buffers of the host-buffer entry points */
int reserve_device_io(b200dpf_ctx *c, size_t key_bytes, size_t out_elems)
{
    const int rc = c->d_keys.reserve((key_bytes + kKeyBytes - 1) / kKeyBytes * kKeyBytes);
    return rc ? rc : c->d_out.reserve(out_elems * sizeof(int32_t));
}

/* Where the kernel finds the live parts of a key. */
struct KeyLayout {
    uint32_t stride_v, root_v;
    int compact;
};
KeyLayout reference_layout() { return KeyLayout{131u, 129u, 0}; }                       /* dpf_wrapper.cu:26-46 */
KeyLayout compact_layout(int depth) { return KeyLayout{2u + 4u * (uint32_t)depth, 1u, 1}; }   /* b200dpf_key_pack */

/* compact form of one key straight into `dst` (b200dpf_key_pack without the checks); the magic is
 * "DPF2", or "DPE4" for an early-terminated key */
constexpr char kMagic[] = "DPF2", kMagicEt[] = "DPE4";

inline void pack_compact(const int32_t *key, uint8_t *dst, int depth, const char *magic = kMagic)
{
    const uint8_t *k = reinterpret_cast<const uint8_t *>(key);
    std::memset(dst, 0, 16);
    std::memcpy(dst, magic, 4);
    dst[4] = (uint8_t)depth;
    std::memcpy(dst + 16, k + 16 * host::SLOT_ROOT, 16);
    uint8_t *o = dst + 32;
    const uint8_t *c1 = k + 16 * host::SLOT_CW1, *c2 = k + 16 * host::SLOT_CW2;
    for (int L = 0; L < depth; L++, o += 64) {
        std::memcpy(o, c1 + 32 * L, 32);
        std::memcpy(o + 32, c2 + 32 * L, 32);
    }
}

/* key number `b` of a batch (null: none) must have been generated for the table's n */
inline int check_key_n(const int32_t *key, int64_t b, int64_t n)
{
    const int64_t kn = key ? host::key_n(key) : -1;
    if (kn == n) return B200DPF_OK;
    return fail(B200DPF_EINVAL, "key %lld was generated for n=%lld, table has n=%lld", (long long)b, (long long)kn, (long long)n);
}

/* key number `b` of a batch must be of the context's kind (standard or early-terminated) and n */
inline int check_key(const b200dpf_ctx *c, const int32_t *key, int64_t b)
{
    if (!c->lane_bits) {
        if (key && host::key_et_n(key) >= 0)
            return fail(B200DPF_EINVAL, "key %lld is an early-terminated key; this context takes standard keys", (long long)b);
        return check_key_n(key, b, c->n);
    }
    const int64_t kn = key ? host::key_et_n(key) : -1;
    if (kn == c->n) return B200DPF_OK;
    if (key && host::key_n(key) >= 0)
        return fail(B200DPF_EINVAL, "key %lld is a standard key; this early-terminated context takes keys of b200dpf_gen_et", (long long)b);
    return fail(B200DPF_EINVAL, "key %lld is not an early-terminated key for n=%lld (its n: %lld)", (long long)b, (long long)c->n,
                (long long)kn);
}

void fill_phase(const SmemLayout &L, int s, PhaseParams *ph)
{
    std::memset(ph, 0, sizeof *ph);
    ph->s = s;
    ph->stack_split = std::min(L.cap_lo, std::max(s - 1, 0));
}

/*
 * One evaluation of <= one leaf-cache-full of keys:
 *   one launch  : [clear result + tickets, build frontier | grid barrier | main]  (+ MAC passes)
 *   legacy      : memset tickets, memset result, frontier kernel, main kernel x passes
 * mode_main is MODE_FUSED (out = [nkeys][entry_size] int32) or MODE_EXPAND
 * (out = [nkeys][n] int32 share vectors).
 */
constexpr int kRetryWithoutCooperativeLaunch = -1000;   /* internal to run_pipeline */

int run_pipeline_chunk(b200dpf_ctx *c, const void *keys_dev, const KeyLayout &kl, int64_t nkeys, int prf, int mode_main,
                       void *out_dev, cudaStream_t stream, bool clear_out, bool want_cache)
{
    const b200dpf_ctx::Knobs &K = c->knobs;
    /* Entries wider than 32 columns: the tree is expanded ONCE by the best-shaped kernel (16
     * columns, NV = 4), which also caches each leaf's low word; every other column is produced by
     * MAC-only passes over that cache.  Without the cache (disabled or lane-split batches) wide
     * entries use one tree expansion per 64 columns. */
    const bool et = c->lane_bits != 0;   /* early-terminated: 32 columns per pass at most */
    const int nv = (mode_main != MODE_FUSED || c->entry_pad <= 16 || want_cache) ? 4 : (c->entry_pad <= 32 || et ? 8 : 16);
    const int passes = mode_main == MODE_FUSED ? (want_cache ? 1 : c->entry_pad / (4 * nv)) : 1;
    /* the kernel modes of this context's kind */
    const int mode_fused = et ? MODE_FUSED_ET : MODE_FUSED, mode_expand = et ? MODE_EXPAND_ET : MODE_EXPAND;
    /* optional variant: the rows of each work item staged into shared memory by cp.async.bulk */
    bool tma_rows = K.tma_rows != 0 && K.one_launch != 0 && c->coop_ok != 0 && mode_main == MODE_FUSED && c->entry_pad == 16 &&
                    prf != B200DPF_PRF_AES128 && nkeys >= 17 && !et;
    const int mode_plain = mode_main == MODE_FUSED ? mode_fused : mode_expand;
    int mode_kernel = tma_rows ? MODE_FUSED_TMA : mode_plain;
    SmemLayout L;
    int rc = smem_layout(c, prf, nv, mode_kernel, &L);
    if (rc) return rc;
    const int64_t warps = (int64_t)L.grid * (L.threads / 32);
    /* keys per warp: a full warp of keys when the batch allows; for small batches the
     * spare lanes take adjacent subtrees of the same keys (single-query latency mode) */
    int kpw_log2 = 5;
    if (K.lane_split != 0)
        while (kpw_log2 > 0 && ((int64_t)1 << (kpw_log2 - 1)) >= nkeys) kpw_log2--;
    int64_t key_groups = (nkeys + ((int64_t)1 << kpw_log2) - 1) >> kpw_log2;

    /* ---- work-item size s and the frontier depth --------------------------------
     * Without a frontier every item re-walks depth-s levels from the root, so items
     * must be big; with one the walk is (almost) free and small items balance the
     * tail. */
    const bool want_frontier = K.frontier != 0;
    int s;
    if (K.subtree_log2 > 0) {
        s = std::min(K.subtree_log2, std::min(c->depth_local, L.s_max));
    } else {
        /* B=512 E=16, frontier on, 1x H100 SXM 80 GB at a 400 W power limit, DPFs/s (run-to-run
         * spread about 3 %); the automatic choice is within the spread of the best fixed s:
         *   AES n=2^20: auto 19.47k; s=4 19.39k, 5 19.77k, 6 19.56k, 7 20.01k, 8 19.56k
         *   AES n=2^16: auto 319.3k; s=4 317.5k, 5 318.1k, 6 318.1k, 7 300.5k
         *   ChaCha n=2^20: auto 19.18k; s=5 18.94k, 6 19.13k, 7 19.19k */
        const int s_cap = want_frontier ? 7 : ((prf == B200DPF_PRF_AES128) ? 8 : 10);
        const int s_floor = want_frontier ? 3 : 5;
        const int64_t items_per_warp = want_frontier ? 24 : 6;
        s = std::min(c->depth_local, std::min(L.s_max, s_cap));
        while (s > s_floor &&
               ((((int64_t)1 << (c->depth_local - s)) * key_groups) >> (5 - kpw_log2)) < items_per_warp * warps)
            s--;
    }
    if (s < 1) s = 1;
    size_t tile_bytes = 0;
    if (tma_rows) {
        /* one tile of 2^s 64-byte rows per warp, after the sibling stack */
        const int warps_blk = L.threads / 32;
        if (K.subtree_log2 <= 0) s = std::min(s, 6);
        tile_bytes = (size_t)warps_blk * ((size_t)64 << s) + 8u * (size_t)warps_blk + 16u;
        if ((size_t)L.off_lo + (size_t)(std::max(s, 7) - 1) * L.level_bytes + tile_bytes > (size_t)L.budget) {
            tma_rows = false;               /* does not fit beside correction words and stack: broadcast loads */
            mode_kernel = mode_plain;
            tile_bytes = 0;
            rc = smem_layout(c, prf, nv, mode_kernel, &L);
            if (rc) return rc;
        }
    }
    const int rel = c->depth_local - s;           /* tree levels between the shard root and the items */
    if (5 - kpw_log2 > rel) {                     /* not enough subtrees to split a warp that far */
        kpw_log2 = 5 - rel;
        key_groups = (nkeys + ((int64_t)1 << kpw_log2) - 1) >> kpw_log2;
    }
    const int spw_log2 = 5 - kpw_log2;
    if (want_cache && kpw_log2 != 5) return fail(B200DPF_ESTATE, "internal: leaf cache planned for a lane-split batch");

    int f_rel = 0;                                /* frontier depth below the shard root (0 = none) */
    if (want_frontier && rel >= 2) {
        const int64_t cap_bytes = (int64_t)K.frontier_mb << 20;
        f_rel = rel;
        while (f_rel > 0 && ((key_groups * (16 << kpw_log2)) << f_rel) > cap_bytes) f_rel--;
        if (f_rel < 2 || f_rel < spw_log2 + 1) f_rel = 0;
    }

    const bool one_launch = K.one_launch != 0 && c->coop_ok != 0;
    const size_t n_main_counters = (size_t)passes * (size_t)key_groups;
    rc = c->d_counters.reserve(n_main_counters * sizeof(uint32_t));
    if (rc) return rc;
    {
        bool grown = false;
        rc = c->d_top_counters.reserve(std::max<size_t>((size_t)key_groups, 64) * sizeof(uint32_t), &grown);
        if (rc) return rc;
        if (grown) c->coop_state_dirty = true;
    }
    if (f_rel > 0) {
        rc = c->d_frontier.reserve(((size_t)key_groups * (16 << kpw_log2)) << f_rel);
        if (rc) return rc;
    }

    rc = wait_last(c, stream);
    if (rc) return rc;

    if (!one_launch || c->coop_state_dirty) {
        CUDA_TRY(cudaMemsetAsync(c->d_top_counters.ptr, 0, c->d_top_counters.cap, stream));
        CUDA_TRY(cudaMemsetAsync(c->d_gridbar.ptr, 0, sizeof(uint32_t), stream));
        c->bar_epoch = 0;
        c->coop_state_dirty = false;
    }
    if (!one_launch) {
        CUDA_TRY(cudaMemsetAsync(c->d_counters.ptr, 0, n_main_counters * sizeof(uint32_t), stream));
        if (mode_main == MODE_FUSED && clear_out)
            CUDA_TRY(cudaMemsetAsync(out_dev, 0, (size_t)nkeys * c->entry_size * sizeof(int32_t), stream));
        c->coop_state_dirty = true;     /* the stand-alone frontier kernel leaves its tickets used */
    }
    c->last_launches = 0;

    /* ---- the tree-top phase (frontier build) ---- */
    EvalParams p;
    size_t smem;
    PhaseParams top;
    std::memset(&top, 0, sizeof top);
    int s_top = 0;
    if (f_rel > 0) {
        SmemLayout LF = L;
        if (!one_launch) {
            rc = smem_layout(c, prf, 4, MODE_FRONTIER, &LF);
            if (rc) return rc;
        }
        s_top = std::max(1, std::min(f_rel - spw_log2, std::min(5, LF.s_max)));
        if (K.top_log2 > 0) {
            s_top = std::max(1, std::min(K.top_log2, std::min(f_rel - spw_log2, LF.s_max)));
        } else if (one_launch && K.balance_top) {
            /* Size of a tree-top item.  The blocks that start at a key group share its 2^(f_rel - s_top)
             * items; an item is (walk to its subtree root) + 2^s_top - 1 node pairs, all sequential.
             * Estimate the phase as rounds x steps x step time, where a step costs the larger of the
             * warps sharing the SM's binding pipe and the latency of one dependent expansion, and take
             * the best size: few long items when blocks are plentiful (one round, few busy warps),
             * more short ones when every warp can be given one.  (AES n=2^20 on 8 shards: s_top 6
             * instead of 5 halves the phase; n=2^14, 16 key groups: 5 stays best.) */
            const int nw = L.threads / 32;
            const double blocks_per_group = std::max(1.0, (double)L.grid / (double)key_groups);
            double best = 1e300;
            for (int cand = 1; cand <= std::min(f_rel - spw_log2, std::min(7, LF.s_max)); cand++) {
                const double tickets = (double)((int64_t)1 << (f_rel - cand)) / (double)(1 << spw_log2) *
                                       std::max(1.0, (double)key_groups / (double)L.grid);
                const double quota = std::ceil(tickets / blocks_per_group);
                const double steps = 0.55 * (c->shard_bits + f_rel - cand) + (double)((1 << cand) - 1);
                const double full_rounds = std::floor(quota / nw), rest = quota - full_rounds * nw;
                const double busy = 330.0, latency = 1500.0;        /* per node pair: pipe slots, dependent-chain latency */
                double t = full_rounds * steps * std::max(nw * busy, latency);
                if (rest > 0) t += steps * std::max(rest * busy, latency);
                if (t < best) {
                    best = t;
                    s_top = cand;
                }
            }
        }
        fill_phase(LF, s_top, &top);
        top.nsub = (uint32_t)1 << (f_rel - s_top);
        top.sub_first = (uint32_t)c->shard_rank << (f_rel - s_top);
        top.walk_first_level = c->depth - 1;
        top.walk_steps = c->shard_bits + f_rel - s_top;
        top.level_base = c->depth_local - f_rel;
        top.counters = c->d_top_counters.ptr;
        if (!one_launch) {
            fill_common(c, LF, s_top, nkeys, kpw_log2, &p, &smem);
            p.keys = reinterpret_cast<const uint4 *>(keys_dev);
            p.key_stride_v = kl.stride_v; p.key_root_v = kl.root_v; p.key_compact = kl.compact;
            p.main = top;
            p.nfront = (uint32_t)1 << f_rel;
            p.frontier_out = reinterpret_cast<uint4 *>(c->d_frontier.ptr);
            CUDA_TRY(launch_eval(prf, 4, MODE_FRONTIER, p, LF.grid, smem, stream));
            c->last_launches++;
        }
    }

    /* ---- the main phase ---- */
    fill_common(c, L, std::max(s, s_top), nkeys, kpw_log2, &p, &smem);
    p.keys = reinterpret_cast<const uint4 *>(keys_dev);
    p.key_stride_v = kl.stride_v; p.key_root_v = kl.root_v; p.key_compact = kl.compact;
    if (tma_rows) {
        p.off_tile = (uint32_t)((smem + 15) & ~(size_t)15);
        p.off_tile_bar = p.off_tile + (uint32_t)((size_t)(L.threads / 32) * ((size_t)64 << s));
        smem = (size_t)p.off_tile + tile_bytes;
    }
    fill_phase(L, s, &p.main);
    p.main.nsub = (uint32_t)1 << rel;
    p.main.sub_first = (uint32_t)c->shard_rank << rel;
    if (f_rel > 0) {
        p.main.frontier_in = reinterpret_cast<const uint4 *>(c->d_frontier.ptr);
        p.nfront = (uint32_t)1 << f_rel;
        p.main.front_shift = rel - f_rel;
        p.main.walk_first_level = c->depth_local - f_rel - 1;
        p.main.walk_steps = rel - f_rel;
    } else {
        p.main.walk_first_level = c->depth - 1;
        p.main.walk_steps = c->depth - s;
    }
    p.main.counters = c->d_counters.ptr;
    if (one_launch) {
        p.fuse_top = 1;
        p.top = top;                      /* nsub == 0: no frontier, the top phase only clears */
        p.frontier_out = reinterpret_cast<uint4 *>(c->d_frontier.ptr);
        if (mode_main == MODE_FUSED && clear_out) {
            p.zero_a = reinterpret_cast<uint32_t *>(out_dev);
            p.zero_a_words = (uint64_t)nkeys * (uint64_t)c->entry_size;
        }
        p.zero_b = c->d_counters.ptr;
        p.zero_b_words = n_main_counters;
        p.rearm = c->d_top_counters.ptr;
        p.rearm_words = (uint32_t)key_groups;
        {
            const uint64_t items = (uint64_t)key_groups * (uint64_t)(top.nsub >> spw_log2);
            p.top_block_quota = K.balance_top ? (uint32_t)std::max<uint64_t>(1, (items + (uint64_t)L.grid - 1) / (uint64_t)L.grid)
                                              : 0x7fffffffu;
        }
        if (K.timing) {
            rc = c->d_timing.reserve((size_t)L.grid * 8 * sizeof(unsigned long long));
            if (rc) return rc;
            CUDA_TRY(cudaMemsetAsync(c->d_timing.ptr, 0, c->d_timing.cap, stream));
            p.timing = c->d_timing.ptr;
        }
        p.grid_bar = c->d_gridbar.ptr;
        c->bar_epoch += (uint32_t)L.grid;
        p.grid_bar_target = c->bar_epoch;
    }
    auto launch_main = [&](int nv_l, int mode_l) -> int {
        const cudaError_t e = launch_eval(prf, nv_l, mode_l, p, L.grid, smem, stream);
        if (e != cudaSuccess) {
            c->coop_state_dirty = true;
            if (e == cudaErrorCooperativeLaunchTooLarge && p.fuse_top) {
                /* this device cannot keep the whole persistent grid resident (a partitioned GPU, say):
                 * nothing of this evaluation has been enqueued yet, so fall back -- for the life of the
                 * context -- to the pipeline of separate launches */
                cudaGetLastError();
                c->coop_ok = 0;
                return kRetryWithoutCooperativeLaunch;
            }
            return fail(B200DPF_ECUDA, "evaluation kernel launch: %s", cudaGetErrorString(e));
        }
        c->last_launches++;
        p.fuse_top = 0;                   /* later passes of this evaluation reuse the frontier */
        return B200DPF_OK;
    };
    if (mode_main == MODE_EXPAND) {
        p.shares = reinterpret_cast<uint32_t *>(out_dev);
        return launch_main(4, mode_expand);
    }
    p.out = reinterpret_cast<uint32_t *>(out_dev);
    if (want_cache) {
        const size_t cache_bytes = (size_t)key_groups * 32u * (size_t)c->n_local * sizeof(uint32_t);
        rc = c->d_leaf_cache.reserve(cache_bytes);
        if (rc) return rc;
        p.leaf_cache = c->d_leaf_cache.ptr;
        p.n_local = (uint64_t)c->n_local;
        p.col_off_v = 0;
        p.col_off = 0;
        p.ncols = (uint32_t)std::min(16, c->entry_size);
        rc = launch_main(4, mode_fused);
        if (rc) return rc;
        MacParams m;
        std::memset(&m, 0, sizeof m);
        m.leaf_cache = p.leaf_cache;
        m.table = p.table;
        m.row_stride_v = p.row_stride_v;
        m.out = p.out;
        m.out_stride = p.out_stride;
        m.nkeys = (int)nkeys;
        m.key_groups = (int)key_groups;
        m.n_local = (uint64_t)c->n_local;
        const bool use_tma = K.mac_tma != 0;
        const int mac_grid = c->sm_count * 2;                      /* register-staged variant */
        const int64_t mac_warps = (int64_t)mac_grid * 8;
        int64_t ranges = std::max<int64_t>(1, (2 * mac_warps + key_groups - 1) / key_groups);
        ranges = std::min<int64_t>(ranges, std::max<int64_t>(1, c->n_local / 64));
        /* TMA variant: one block per SM; a block takes 8 key groups x one position range */
        const int64_t kg_blocks = (key_groups + 7) / 8;
        int64_t tr = std::max<int64_t>(1, (2 * (int64_t)c->sm_count + kg_blocks - 1) / kg_blocks);
        tr = std::min<int64_t>(tr, std::max<int64_t>(1, c->n_local / 256));
        for (int blk = 0; blk * 64 < c->entry_size; blk++) {       /* 64-column slices of the rows */
            m.col_off_v = (uint32_t)(blk * 16);
            m.col_off = (uint32_t)(blk * 64);
            m.ncols = (uint32_t)std::min(64, c->entry_size - blk * 64);
            m.col_skip = blk == 0 ? 16u : 0u;                      /* columns 0..15 came from the fused pass */
            if (m.ncols <= m.col_skip) continue;
            if (use_tma) {
                m.ranges_per_group = (uint32_t)tr;
                CUDA_TRY(launch_mac_tma(m, c->sm_count, stream));
            } else {
                m.ranges_per_group = (uint32_t)ranges;
                CUDA_TRY(launch_mac(16, m, mac_grid, stream));
            }
            c->last_launches++;
        }
        return B200DPF_OK;
    }
    for (int pass = 0; pass < passes; pass++) {
        p.col_off_v = (uint32_t)(pass * nv);
        p.col_off = (uint32_t)(pass * 4 * nv);
        p.ncols = (uint32_t)std::max(0, std::min(4 * nv, c->entry_size - pass * 4 * nv));
        if (p.ncols == 0) break;
        p.main.counters = c->d_counters.ptr + (size_t)pass * key_groups;
        rc = launch_main(nv, mode_kernel);
        if (rc) return rc;
    }
    return B200DPF_OK;
}

/*
 * One evaluation.  Wide entries whose leaf cache (nkeys x n_local x 4 bytes) would exceed the cap
 * are evaluated in batch chunks that fit -- the cache is what makes columns beyond the first 16
 * cost a MAC pass instead of a tree expansion, so shrinking the chunk beats dropping the cache.
 */
int run_pipeline(b200dpf_ctx *c, const void *keys_dev, const KeyLayout &kl, int64_t nkeys, int prf, int mode_main,
                 void *out_dev, cudaStream_t stream, bool clear_out = true)
{
    const b200dpf_ctx::Knobs &K = c->knobs;
    int rc = B200DPF_OK;
    int launches = 0;
    const bool wide = mode_main == MODE_FUSED && c->entry_pad > 32 && nkeys >= 17 && K.leaf_cache != 0;
    const size_t per_group = 32u * (size_t)c->n_local * sizeof(uint32_t);
    const size_t cap = (size_t)std::max(K.leaf_cache_mb, 1) << 20;
    if (!wide || per_group > cap) {
        /* not a cached evaluation (or one key group alone overflows the cap: re-expand per 64 columns) */
        rc = run_pipeline_chunk(c, keys_dev, kl, nkeys, prf, mode_main, out_dev, stream, clear_out, false);
        if (rc == kRetryWithoutCooperativeLaunch)
            rc = run_pipeline_chunk(c, keys_dev, kl, nkeys, prf, mode_main, out_dev, stream, clear_out, false);
        launches = c->last_launches;
    } else {
        const int64_t groups_per_chunk = (int64_t)std::max<size_t>(1, cap / per_group);
        const int64_t chunk = groups_per_chunk * 32;
        for (int64_t k0 = 0; k0 < nkeys && rc == B200DPF_OK; k0 += chunk) {
            const int64_t kn = std::min(chunk, nkeys - k0);
            const char *kp = reinterpret_cast<const char *>(keys_dev) + (size_t)k0 * kl.stride_v * 16u;
            char *op = reinterpret_cast<char *>(out_dev) + (size_t)k0 * c->entry_size * sizeof(int32_t);
            /* a ragged tail below 17 keys would be lane-split, which the cache layout excludes */
            rc = run_pipeline_chunk(c, kp, kl, kn, prf, mode_main, op, stream, clear_out, kn >= 17);
            if (rc == kRetryWithoutCooperativeLaunch)
                rc = run_pipeline_chunk(c, kp, kl, kn, prf, mode_main, op, stream, clear_out, kn >= 17);
            launches += c->last_launches;
        }
    }
    c->last_launches = launches;
    return rc ? rc : mark_last(c, stream);
}

int run_eval(b200dpf_ctx *c, const void *keys_dev, int64_t nkeys, int prf, void *out_dev, cudaStream_t stream)
{
    return run_pipeline(c, keys_dev, reference_layout(), nkeys, prf, MODE_FUSED, out_dev, stream);
}

bool is_pinned_host(const void *ptr)
{
    cudaPointerAttributes attr;
    const bool yes = cudaPointerGetAttributes(&attr, ptr) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    return yes;
}

/* Copy `elems` results from the context's d_out into the caller's host buffer `out` and wait for them;
 * pageable memory is staged through the pinned h_out so the copy is a real asynchronous DMA. */
int download_out(b200dpf_ctx *c, int32_t *out, bool out_pinned, size_t elems)
{
    int32_t *dst = out;
    if (!out_pinned) {
        const int rc = reserve_host_out(c, elems);
        if (rc) return rc;
        dst = c->h_out.ptr;
    }
    CUDA_TRY(cudaMemcpyAsync(dst, c->d_out.ptr, elems * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (dst != out) std::memcpy(out, dst, elems * sizeof(int32_t));
    return B200DPF_OK;
}

/* The evaluation of keys already enqueued for upload into d_keys, timed, and its results into `out`. */
int eval_tail(b200dpf_ctx *c, const KeyLayout &kl, int64_t nkeys, int prf, int32_t *out)
{
    CUDA_TRY(cudaEventRecord(c->ev_t0, c->stream));
    const int rc = run_pipeline(c, c->d_keys.ptr, kl, nkeys, prf, MODE_FUSED, c->d_out.ptr, c->stream);
    if (rc) return rc;
    CUDA_TRY(cudaEventRecord(c->ev_t1, c->stream));
    c->timed = true;
    return download_out(c, out, is_pinned_host(out), (size_t)nkeys * c->entry_size);
}

int check_eval_args(const b200dpf_ctx *c, const void *keys, int64_t nkeys, int prf, const void *out)
{
    if (!c) return fail(B200DPF_EINVAL, "null context");
    if (!c->d_table.ptr && !c->multi) return fail(B200DPF_ESTATE, "context has no table");
    if (c->bins) return fail(B200DPF_ESTATE, "grouped context: use b200dpf_group_eval");
    if (!keys || !out) return fail(B200DPF_EINVAL, "null buffer");
    if (nkeys < 1 || nkeys > (int64_t)1 << 24) return fail(B200DPF_EINVAL, "nkeys=%lld out of range", (long long)nkeys);
    if (prf < B200DPF_PRF_DUMMY || prf > B200DPF_PRF_AES128) return fail(B200DPF_EINVAL, "unknown prf id %d", prf);
    return B200DPF_OK;
}

/* Check that `device` exists and make it current for as long as `guard` lives; `cpu_hint` completes the
 * message on a machine without CUDA devices. */
int open_device(int device, const char *cpu_hint, std::optional<DeviceGuard> *guard)
{
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return fail(B200DPF_ECUDA, "no CUDA device available (%s)", cpu_hint);
    if (device < 0 || device >= ndev) return fail(B200DPF_EINVAL, "device %d out of range (have %d)", device, ndev);
    guard->emplace(device);
    if (!(*guard)->ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", device);
    return B200DPF_OK;
}

/* The set-up both create functions share: a context on `device`, current while `guard` lives, with the
 * device's properties, its stream and events, the grid-barrier word, the shared-memory base and the AES
 * tables.  With `read_env` the tuning knobs start from the B200DPF_* environment variables. */
int ctx_open(int device, bool read_env, std::optional<DeviceGuard> *guard, std::unique_ptr<b200dpf_ctx> *out)
{
    int rc = open_device(device, "this engine has no CPU fallback", guard);
    if (rc) return rc;
    std::unique_ptr<b200dpf_ctx> c(new (std::nothrow) b200dpf_ctx());
    if (!c) return fail(B200DPF_ENOMEM, "out of host memory");
    c->device = device;
    CUDA_TRY(cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device));
    CUDA_TRY(cudaDeviceGetAttribute(&c->coop_ok, cudaDevAttrCooperativeLaunch, device));
    CUDA_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreate(&c->ev_t0));
    CUDA_TRY(cudaEventCreate(&c->ev_t1));
    rc = c->d_gridbar.reserve(sizeof(uint32_t));
    if (rc) return rc;
    if (read_env) {
        /* the environment is consulted here and nowhere else (b200dpf_ctx_set_option changes a
         * live context) */
        b200dpf_ctx::Knobs &K = c->knobs;
        K.leaf_cache = env_int("B200DPF_LEAF_CACHE", K.leaf_cache);
        K.leaf_cache_mb = env_int("B200DPF_LEAF_CACHE_MB", K.leaf_cache_mb);
        K.lane_split = env_int("B200DPF_LANE_SPLIT", K.lane_split);
        K.frontier = env_int("B200DPF_FRONTIER", K.frontier);
        K.frontier_mb = env_int("B200DPF_FRONTIER_MB", K.frontier_mb);
        K.subtree_log2 = env_int("B200DPF_S", K.subtree_log2);
        K.mac_tma = env_int("B200DPF_MAC_TMA", K.mac_tma);
        K.one_launch = env_int("B200DPF_ONE_LAUNCH", K.one_launch);
        K.balance_top = env_int("B200DPF_BALANCE_TOP", K.balance_top);
        K.timing = env_int("B200DPF_TIMING", K.timing);
        K.top_log2 = env_int("B200DPF_TOP_LOG2", K.top_log2);
        K.tma_rows = env_int("B200DPF_TMA_ROWS", K.tma_rows);
    }
    CUDA_TRY(probe_dynamic_smem_base(&c->smem_base, c->stream));
    CUDA_TRY(upload_aes_table(host::aes_te0()));
    *out = std::move(c);
    return B200DPF_OK;
}

/* Run gen_one(i) for every i < count on `nthreads` threads (0: one per hardware thread); false when any
 * call failed. */
template <class GenOne>
bool gen_parallel(int64_t count, int nthreads, GenOne gen_one)
{
    if (nthreads <= 0) nthreads = (int)std::max(1u, std::thread::hardware_concurrency());
    nthreads = (int)std::min<int64_t>(nthreads, std::max<int64_t>(count, 1));
    std::vector<int> rcs((size_t)nthreads, 0);
    auto work = [&](int t) {
        for (int64_t i = t; i < count; i += nthreads)
            if (gen_one(i)) rcs[(size_t)t] = -1;
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < nthreads; t++) pool.emplace_back(work, t);
    work(0);
    for (auto &th : pool) th.join();
    return std::find(rcs.begin(), rcs.end(), -1) == rcs.end();
}

}  // namespace

/* multi-device contexts (defined at the end of this file) */
static b200dpf_ctx *multi_first(b200dpf_ctx *root);
static int multi_last_launches(const b200dpf_ctx *root);
static int multi_set_option(b200dpf_ctx *root, const char *name, int value);
static int multi_eval_host(b200dpf_ctx *root, const void *keys, size_t key_stride_bytes, const KeyLayout &kl, int64_t nkeys,
                           int prf, int32_t *out);

extern "C" {

const char *b200dpf_version(void) { return "b200dpf 0.1.0 sm_90a"; }

const char *b200dpf_last_error(void) { return g_err; }

int b200dpf_gen(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf,
                int32_t *key_a, int32_t *key_b)
{
    if (!key_a || !key_b) return fail(B200DPF_EINVAL, "null key buffer");
    uint32_t seed32 = 0;
    for (size_t i = 0; i < 4 && i < seed_len && seed; i++) seed32 |= (uint32_t)seed[i] << (8 * i);
    if (host::gen(alpha, n, seed32, prf, key_a, key_b) != 0)
        return fail(B200DPF_EINVAL, "gen: need power-of-two n >= 2, 0 <= alpha < n, valid prf (alpha=%lld n=%lld prf=%d)",
                    (long long)alpha, (long long)n, prf);
    return B200DPF_OK;
}

int b200dpf_gen_secure(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf,
                       int32_t *key_a, int32_t *key_b)
{
    if (!key_a || !key_b) return fail(B200DPF_EINVAL, "null key buffer");
    if (!seed || seed_len < 44) return fail(B200DPF_EINVAL, "gen_secure needs at least 44 bytes of seed (got %zu)", seed_len);
    if (host::gen_secure(alpha, n, seed, prf, key_a, key_b) != 0)
        return fail(B200DPF_EINVAL, "gen_secure: need power-of-two n >= 2, 0 <= alpha < n, valid prf (alpha=%lld n=%lld prf=%d)",
                    (long long)alpha, (long long)n, prf);
    return B200DPF_OK;
}

int b200dpf_gen_batch(const int64_t *alphas, const uint32_t *seeds32, int64_t count, int64_t n, int prf,
                      int nthreads, int32_t *keys_a, int32_t *keys_b)
{
    if (!alphas || !seeds32 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad gen_batch argument");
    if (!gen_parallel(count, nthreads, [&](int64_t i) {
            return host::gen(alphas[i], n, seeds32[i], prf, keys_a + i * host::KEY_WORDS, keys_b + i * host::KEY_WORDS);
        }))
        return fail(B200DPF_EINVAL, "gen_batch: invalid alpha/n/prf in batch");
    return B200DPF_OK;
}

int b200dpf_gen_batch_secure(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                             int nthreads, int32_t *keys_a, int32_t *keys_b)
{
    if (!alphas || !seeds44 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad gen_batch_secure argument");
    if (!gen_parallel(count, nthreads, [&](int64_t i) {
            return host::gen_secure(alphas[i], n, seeds44 + 44 * i, prf, keys_a + i * host::KEY_WORDS, keys_b + i * host::KEY_WORDS);
        }))
        return fail(B200DPF_EINVAL, "gen_batch_secure: invalid alpha/n/prf in batch");
    return B200DPF_OK;
}

int b200dpf_gen_batch_gpu(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int device,
                          int32_t *keys_a, int32_t *keys_b)
{
    if (!alphas || !seeds44 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad gen_batch_gpu argument");
    if (n < 2 || n > ((int64_t)1 << 32) || (n & (n - 1)) != 0) return fail(B200DPF_EINVAL, "n=%lld must be a power of two in [2, 2^32]", (long long)n);
    if (prf < B200DPF_PRF_DUMMY || prf > B200DPF_PRF_AES128) return fail(B200DPF_EINVAL, "unknown prf id %d", prf);
    for (int64_t i = 0; i < count; i++)
        if (alphas[i] < 0 || alphas[i] >= n) return fail(B200DPF_EINVAL, "gen_batch_gpu: alpha[%lld]=%lld out of range", (long long)i, (long long)alphas[i]);
    if (count == 0) return B200DPF_OK;
    std::optional<DeviceGuard> guard;
    int rc = open_device(device, "use b200dpf_gen_batch_secure on the CPU", &guard);
    if (rc) return rc;
    const size_t key_bytes = (size_t)count * kKeyBytes;
    DeviceBuffer<int64_t> d_alphas;
    DeviceBuffer<uint8_t> d_seeds;
    DeviceBuffer<uint32_t> d_te0;
    DeviceBuffer<uint4> d_a, d_b;
    rc = d_alphas.reserve((size_t)count * sizeof(int64_t));
    if (!rc) rc = d_seeds.reserve((size_t)count * 44);
    if (!rc) rc = d_te0.reserve(256 * sizeof(uint32_t));
    if (!rc) rc = d_a.reserve(key_bytes);
    if (!rc) rc = d_b.reserve(key_bytes);
    if (rc) return rc;
    cudaError_t e = cudaMemcpy(d_alphas.ptr, alphas, (size_t)count * sizeof(int64_t), cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(d_seeds.ptr, seeds44, (size_t)count * 44, cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(d_te0.ptr, host::aes_te0(), 256 * sizeof(uint32_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
        e = launch_keygen(prf, d_alphas.ptr, d_seeds.ptr, count, ilog2(n), (uint64_t)n, d_te0.ptr, d_a.ptr, d_b.ptr, nullptr);
    if (e == cudaSuccess) e = cudaMemcpy(keys_a, d_a.ptr, key_bytes, cudaMemcpyDefault);      /* host or device destination */
    if (e == cudaSuccess) e = cudaMemcpy(keys_b, d_b.ptr, key_bytes, cudaMemcpyDefault);
    if (e != cudaSuccess) return fail(B200DPF_ECUDA, "gen_batch_gpu: %s", cudaGetErrorString(e));
    return B200DPF_OK;
}

int b200dpf_eval_cpu(const int32_t *key, int prf, int32_t *out_n)
{
    if (!key || !out_n) return fail(B200DPF_EINVAL, "null buffer");
    if (host::eval_cpu(key, prf, out_n) != 0) return fail(B200DPF_EINVAL, "eval_cpu: malformed key or prf id");
    return B200DPF_OK;
}

size_t b200dpf_key_packed_size(int depth) { return depth >= 1 && depth <= 32 ? (size_t)32 + 64u * (size_t)depth : 0; }

int b200dpf_key_pack(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    if (!key || !out) return fail(B200DPF_EINVAL, "null buffer");
    const int depth = host::key_depth(key);
    if (depth < 1 || host::key_n(key) < 0) return fail(B200DPF_EINVAL, "key_pack: malformed key");
    const size_t need = b200dpf_key_packed_size(depth);
    if (out_cap < need) return fail(B200DPF_EINVAL, "key_pack: need %zu bytes, have %zu", need, out_cap);
    pack_compact(key, out, depth);
    if (written) *written = need;
    return B200DPF_OK;
}

int b200dpf_key_unpack(const uint8_t *in, size_t in_len, int32_t *key)
{
    if (!in || !key) return fail(B200DPF_EINVAL, "null buffer");
    if (in_len < 32 || std::memcmp(in, "DPF2", 4) != 0) return fail(B200DPF_EINVAL, "key_unpack: bad header");
    const int depth = in[4];
    bool pad_zero = true;
    for (int i = 5; i < 16; i++) pad_zero = pad_zero && in[i] == 0;
    if (depth < 1 || depth > 32 || !pad_zero || in_len != b200dpf_key_packed_size(depth))
        return fail(B200DPF_EINVAL, "key_unpack: depth %d does not match %zu bytes", depth, in_len);
    std::memset(key, 0, sizeof(int32_t) * host::KEY_WORDS);
    uint8_t *k = reinterpret_cast<uint8_t *>(key);
    k[16 * host::SLOT_DEPTH] = (uint8_t)depth;
    std::memcpy(k + 16 * host::SLOT_ROOT, in + 16, 16);
    for (int L = 0; L < depth; L++) {
        const uint8_t *o = in + 32 + 64 * L;
        std::memcpy(k + 16 * (host::SLOT_CW1 + 2 * L), o, 32);
        std::memcpy(k + 16 * (host::SLOT_CW2 + 2 * L), o + 32, 32);
    }
    const uint64_t n = (uint64_t)1 << depth;
    std::memcpy(k + 16 * host::SLOT_N, &n, 8);
    return B200DPF_OK;
}

int64_t b200dpf_key_n(const int32_t *key) { return key ? host::key_n(key) : -1; }
int b200dpf_key_depth(const int32_t *key) { return key ? host::key_depth(key) : -1; }

/* ---- early-terminated keys ---- */

int b200dpf_gen_et(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf, int32_t *key_a, int32_t *key_b)
{
    if (!key_a || !key_b) return fail(B200DPF_EINVAL, "null key buffer");
    if (!seed || seed_len < 44) return fail(B200DPF_EINVAL, "gen_et needs at least 44 bytes of seed (got %zu)", seed_len);
    if (host::gen_et(alpha, n, seed, prf, key_a, key_b) != 0)
        return fail(B200DPF_EINVAL, "gen_et: need power-of-two n in [8, 2^31], 0 <= alpha < n, valid prf (alpha=%lld n=%lld prf=%d)",
                    (long long)alpha, (long long)n, prf);
    return B200DPF_OK;
}

int b200dpf_gen_batch_et(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int nthreads,
                         int32_t *keys_a, int32_t *keys_b)
{
    if (!alphas || !seeds44 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad gen_batch_et argument");
    if (!gen_parallel(count, nthreads, [&](int64_t i) {
            return host::gen_et(alphas[i], n, seeds44 + 44 * i, prf, keys_a + i * host::KEY_WORDS, keys_b + i * host::KEY_WORDS);
        }))
        return fail(B200DPF_EINVAL, "gen_batch_et: invalid alpha/n/prf in batch");
    return B200DPF_OK;
}

int b200dpf_eval_cpu_et(const int32_t *key, int prf, int32_t *out_n)
{
    if (!key || !out_n) return fail(B200DPF_EINVAL, "null buffer");
    if (host::key_et_n(key) < 0) return fail(B200DPF_EINVAL, "eval_cpu_et: not an early-terminated key");
    if (host::eval_cpu_et(key, prf, out_n) != 0) return fail(B200DPF_EINVAL, "eval_cpu_et: unknown prf id %d", prf);
    return B200DPF_OK;
}

int b200dpf_key_pack_et(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    if (!key || !out) return fail(B200DPF_EINVAL, "null buffer");
    const int depth = host::key_et_depth(key);
    if (depth < 1 || host::key_et_n(key) < 0) return fail(B200DPF_EINVAL, "key_pack_et: not an early-terminated key");
    const size_t need = b200dpf_key_packed_size(depth);
    if (out_cap < need) return fail(B200DPF_EINVAL, "key_pack_et: need %zu bytes, have %zu", need, out_cap);
    pack_compact(key, out, depth, kMagicEt);
    if (written) *written = need;
    return B200DPF_OK;
}

int b200dpf_key_unpack_et(const uint8_t *in, size_t in_len, int32_t *key)
{
    if (!in || !key) return fail(B200DPF_EINVAL, "null buffer");
    if (in_len < 32 || std::memcmp(in, kMagicEt, 4) != 0) return fail(B200DPF_EINVAL, "key_unpack_et: bad header");
    const int depth = in[4];
    bool pad_zero = true;
    for (int i = 5; i < 16; i++) pad_zero = pad_zero && in[i] == 0;
    if (depth < 1 || depth > host::ET_MAX_DEPTH || !pad_zero || in_len != b200dpf_key_packed_size(depth))
        return fail(B200DPF_EINVAL, "key_unpack_et: depth %d does not match %zu bytes", depth, in_len);
    std::memset(key, 0, sizeof(int32_t) * host::KEY_WORDS);
    uint8_t *k = reinterpret_cast<uint8_t *>(key);
    k[16 * host::SLOT_DEPTH] = (uint8_t)depth;
    k[16 * host::SLOT_DEPTH + 4] = (uint8_t)host::ET_LOG2_ROWS_PER_LEAF;
    std::memcpy(k + 16 * host::SLOT_ROOT, in + 16, 16);
    for (int L = 0; L < depth; L++) {
        const uint8_t *o = in + 32 + 64 * L;
        std::memcpy(k + 16 * (host::SLOT_CW1 + 2 * L), o, 32);
        std::memcpy(k + 16 * (host::SLOT_CW2 + 2 * L), o + 32, 32);
    }
    const uint64_t n = (uint64_t)1 << (depth + host::ET_LOG2_ROWS_PER_LEAF);
    std::memcpy(k + 16 * host::SLOT_N, &n, 8);
    return B200DPF_OK;
}

}  // extern "C"

/* b200dpf_create (lane_bits = 0) and b200dpf_create_et (lane_bits = 2: 2^lane_bits rows per leaf) */
static int create_impl(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int device, int shard_rank,
                       int shard_count, int lane_bits)
{
    if (!out) return fail(B200DPF_EINVAL, "null ctx out pointer");
    *out = nullptr;
    if (!table) return fail(B200DPF_EINVAL, "null table");
    const int64_t n_min = (int64_t)2 << lane_bits;
    if (n < n_min || n > ((int64_t)1 << 31) || (n & (n - 1)) != 0)
        return fail(B200DPF_EINVAL, "table size n=%lld must be a power of two in [%lld, 2^31]", (long long)n, (long long)n_min);
    if (entry_size < 1 || entry_size > 4096) return fail(B200DPF_EINVAL, "entry_size=%d out of range [1,4096]", entry_size);
    if (shard_count < 1 || (shard_count & (shard_count - 1)) != 0 || (int64_t)shard_count > n / n_min ||
        shard_rank < 0 || shard_rank >= shard_count)
        return fail(B200DPF_EINVAL, "bad shard %d of %d for n=%lld", shard_rank, shard_count, (long long)n);

    std::optional<DeviceGuard> guard;
    std::unique_ptr<b200dpf_ctx> c;
    int rc = ctx_open(device, true, &guard, &c);
    if (rc) return rc;
    c->n = n;
    c->lane_bits = lane_bits;
    c->depth = ilog2(n) - lane_bits;   /* the tree is over leaves */
    c->entry_size = entry_size;
    /* rows padded to what one pass reads: 16, 32 or a multiple of 64 int32 */
    c->entry_pad = entry_size <= 16 ? 16 : (entry_size <= 32 ? 32 : ((entry_size + 63) & ~63));
    c->shard_rank = shard_rank;
    c->shard_count = shard_count;
    c->shard_bits = ilog2(shard_count);
    c->n_local = n / shard_count;
    c->depth_local = c->depth - c->shard_bits;

    /* Table: gather this shard's rows (natural indices j*G + bitrev_g(rank)),
     * then permute on the device into breadth-first leaf order, padded to
     * 64-byte rows.  dpf_wrapper.cu:103-115 does the analogous reorder on the
     * host with one ATen call per element.  On an early-terminated context the
     * same is done to runs of 2^lane_bits rows, one leaf each. */
    {   /* a device-resident table may still be being written on the caller's stream (e.g. a dtype
         * cast enqueued just before this call): our copy runs on a private non-blocking stream,
         * so wait for the producing device first */
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, table) == cudaSuccess &&
            (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) {
            if (attr.device != device) cudaSetDevice(attr.device);
            const cudaError_t es = cudaDeviceSynchronize();
            if (attr.device != device) cudaSetDevice(device);
            CUDA_TRY(es);
        }
        cudaGetLastError();
    }
    const size_t row_bytes = (size_t)entry_size * sizeof(int32_t);
    const size_t stage_bytes = (size_t)c->n_local * row_bytes;
    const size_t leaf_bytes = row_bytes << lane_bits;            /* one leaf's rows */
    const int64_t leaves_local = c->n_local >> lane_bits;
    const size_t table_bytes = (size_t)c->n_local * (size_t)c->entry_pad * sizeof(int32_t);
    DeviceBuffer<int32_t> d_stage;
    rc = d_stage.reserve(stage_bytes);
    if (rc) return rc;
    cudaError_t e = cudaSuccess;
    if (shard_count == 1) {
        e = cudaMemcpyAsync(d_stage.ptr, table, stage_bytes, cudaMemcpyDefault, c->stream);
    } else {
        const int32_t *src = table + ((size_t)bitrev_host((uint32_t)shard_rank, c->shard_bits) << lane_bits) * entry_size;
        cudaPointerAttributes attr;
        const bool on_device = cudaPointerGetAttributes(&attr, table) == cudaSuccess &&
                               (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
        cudaGetLastError();
        if (on_device) {
            e = cudaMemcpy2DAsync(d_stage.ptr, leaf_bytes, src, leaf_bytes * shard_count, leaf_bytes, (size_t)leaves_local,
                                  cudaMemcpyDefault, c->stream);
        } else {
            std::vector<int32_t> gathered((size_t)c->n_local * entry_size);
            const size_t leaf_words = (size_t)entry_size << lane_bits;
            for (int64_t j = 0; j < leaves_local; j++)
                std::memcpy(gathered.data() + (size_t)j * leaf_words, src + (size_t)j * shard_count * leaf_words, leaf_bytes);
            e = cudaMemcpyAsync(d_stage.ptr, gathered.data(), stage_bytes, cudaMemcpyHostToDevice, c->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        }
    }
    CUDA_TRY(e);
    rc = c->d_table.reserve(table_bytes);
    if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_table.ptr, 0, table_bytes, c->stream));
    if (lane_bits)
        CUDA_TRY(launch_permute_table_et(d_stage.ptr, c->d_table.ptr, (uint64_t)c->n_local, c->depth_local, entry_size,
                                         c->entry_pad, c->sm_count, c->stream));
    else
        CUDA_TRY(launch_permute_table(d_stage.ptr, c->d_table.ptr, (uint64_t)c->n_local, c->depth_local, entry_size,
                                      c->entry_pad, c->sm_count, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    d_stage.release();

    /* Like the reference's eval_init (dpf_wrapper.cu:120-129), set up everything a default batch
     * (512 keys) needs now, so the first evaluation pays neither allocations nor lazy module
     * loading: device key/result/ticket buffers, pinned staging, launch layouts of every PRF. */
    const size_t b0 = B200DPF_DEFAULT_BATCH_SIZE;
    rc = reserve_device_io(c.get(), b0 * kKeyBytes, b0 * entry_size);
    if (!rc) rc = reserve_host_keys(c.get(), b0 * kKeyBytes);
    if (!rc) rc = reserve_host_out(c.get(), b0 * entry_size);
    if (rc) return rc;
    const int nv0 = c->entry_pad <= 16 ? 4 : (c->entry_pad <= 32 ? 8 : 4);
    SmemLayout tmp;
    for (int prf = 0; prf < 4; prf++) {
        smem_layout(c.get(), prf, nv0, lane_bits ? MODE_FUSED_ET : MODE_FUSED, &tmp);
        smem_layout(c.get(), prf, 4, MODE_FRONTIER, &tmp);
    }
    *out = c.release();
    return B200DPF_OK;
}

extern "C" {

int b200dpf_create(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int device,
                   int shard_rank, int shard_count)
{
    return create_impl(out, table, n, entry_size, device, shard_rank, shard_count, 0);
}

int b200dpf_create_et(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int device,
                      int shard_rank, int shard_count)
{
    return create_impl(out, table, n, entry_size, device, shard_rank, shard_count, host::ET_LOG2_ROWS_PER_LEAF);
}

int b200dpf_ctx_rows_per_leaf(const b200dpf_ctx *c) { return c ? 1 << c->lane_bits : -1; }

int b200dpf_destroy(b200dpf_ctx *c)
{
    if (!c) return B200DPF_OK;
    DeviceGuard guard(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    delete c;
    return B200DPF_OK;
}

/* Host buffers in and out: keys (either layout) -> pinned staging if pageable -> H2D, the
 * evaluation, D2H, one stream synchronisation. */
static int eval_host(b200dpf_ctx *c, const void *keys, size_t key_bytes, const KeyLayout &kl, int64_t nkeys, int prf,
                     int32_t *out)
{
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    int rc = reserve_device_io(c, key_bytes, (size_t)nkeys * c->entry_size);
    if (rc) return rc;
    /* pageable host memory goes through the context's pinned staging so both copies are real
     * asynchronous DMA transfers; already-pinned buffers (ours or the caller's) are used as is */
    const void *src = keys;
    if (!is_pinned_host(keys)) {
        rc = reserve_host_keys(c, key_bytes);
        if (rc) return rc;
        std::memcpy(c->h_keys.ptr, keys, key_bytes);
        src = c->h_keys.ptr;
    }
    /* the previous evaluation may have run on a caller's stream: the staging copy below must not
     * overtake it (run_pipeline orders the kernels, this orders the H2D) */
    rc = wait_last(c, c->stream);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_keys.ptr, src, key_bytes, cudaMemcpyHostToDevice, c->stream));
    return eval_tail(c, kl, nkeys, prf, out);
}

static int eval_gather_impl(b200dpf_ctx *c, const int32_t *const *keys, int64_t nkeys, int prf, int32_t *out, bool validate);

int b200dpf_eval(b200dpf_ctx *c, const int32_t *keys, int64_t nkeys, int prf, int32_t *out)
{
    int rc = check_eval_args(c, keys, nkeys, prf, out);
    if (rc) return rc;
    for (int64_t b = 0; b < nkeys; b++)
        if ((rc = check_key(c, keys + b * host::KEY_WORDS, b))) return rc;
    if (!is_pinned_host(keys)) {
        /* pageable keys have to be staged by the CPU anyway: stage only their live 32 + 64*depth bytes
         * (44 % of a key at n = 2^14, 63 % at 2^20) and let the DMA of a chunk overlap the next one */
        std::vector<const int32_t *> ptrs((size_t)nkeys);
        for (int64_t b = 0; b < nkeys; b++) ptrs[(size_t)b] = keys + b * host::KEY_WORDS;
        return eval_gather_impl(c, ptrs.data(), nkeys, prf, out, false);   /* validated just above */
    }
    if (c->multi) return multi_eval_host(c, keys, host::KEY_WORDS * sizeof(int32_t), reference_layout(), nkeys, prf, out);
    return eval_host(c, keys, (size_t)nkeys * host::KEY_WORDS * sizeof(int32_t), reference_layout(), nkeys, prf, out);
}

/* keys given as pointers: gather the live parts into pinned staging in the compact layout (validating them
 * if asked), upload chunk by chunk while gathering, evaluate, copy back */
static int eval_gather_impl(b200dpf_ctx *c, const int32_t *const *keys, int64_t nkeys, int prf, int32_t *out, bool validate)
{
    b200dpf_ctx *c0 = c->multi ? multi_first(c) : c;
    DeviceGuard guard(c0->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c0->device);
    const size_t stride = b200dpf_key_packed_size(c->depth);
    const size_t key_bytes = (size_t)nkeys * stride;
    int rc = reserve_host_keys(c0, key_bytes);
    if (rc) return rc;
    uint8_t *stage = reinterpret_cast<uint8_t *>(c0->h_keys.ptr);
    if (!c->multi) {
        rc = reserve_device_io(c, key_bytes, (size_t)nkeys * c->entry_size);
        if (rc) return rc;
        rc = wait_last(c, c->stream);
        if (rc) return rc;
    }
    /* pack a chunk into pinned staging, start its DMA, pack the next: the copy engine works while
     * the host gathers (the reference converts all 512 keys, then issues one blocking cudaMemcpy);
     * a multi-device context uploads from the whole staged batch instead */
    const int64_t chunk = 64;
    for (int64_t b0 = 0; b0 < nkeys; b0 += chunk) {
        const int64_t b1 = std::min(nkeys, b0 + chunk);
        for (int64_t b = b0; b < b1; b++) {
            /* validated here, while the key's cache lines are being read anyway (one pass over 512 scattered
             * 2 KiB keys instead of two); copies already issued for earlier chunks are harmless on failure */
            if (validate && (rc = check_key(c, keys[b], b))) return rc;
            pack_compact(keys[b], stage + (size_t)b * stride, c->depth, c->lane_bits ? kMagicEt : kMagic);
        }
        if (!c->multi)
            CUDA_TRY(cudaMemcpyAsync(reinterpret_cast<uint8_t *>(c->d_keys.ptr) + (size_t)b0 * stride, stage + (size_t)b0 * stride,
                                     (size_t)(b1 - b0) * stride, cudaMemcpyHostToDevice, c->stream));
    }
    if (c->multi) return multi_eval_host(c, stage, stride, compact_layout(c->depth), nkeys, prf, out);
    return eval_tail(c, compact_layout(c->depth), nkeys, prf, out);
}

int b200dpf_eval_gather(b200dpf_ctx *c, const int32_t *const *keys, int64_t nkeys, int prf, int32_t *out)
{
    int rc = check_eval_args(c, keys, nkeys, prf, out);
    if (rc) return rc;
    return eval_gather_impl(c, keys, nkeys, prf, out, true);
}

int b200dpf_eval_packed(b200dpf_ctx *c, const uint8_t *packed, int64_t nkeys, int prf, int32_t *out)
{
    int rc = check_eval_args(c, packed, nkeys, prf, out);
    if (rc) return rc;
    const size_t stride = b200dpf_key_packed_size(c->depth);
    for (int64_t b = 0; b < nkeys; b++) {
        const uint8_t *k = packed + (size_t)b * stride;
        if (std::memcmp(k, c->lane_bits ? kMagicEt : kMagic, 4) != 0 || k[4] != (uint8_t)c->depth)
            return fail(B200DPF_EINVAL, "packed key %lld: bad header or depth %d, table has depth %d (n=%lld)", (long long)b,
                        (int)k[4], c->depth, (long long)c->n);
    }
    if (c->multi) return multi_eval_host(c, packed, stride, compact_layout(c->depth), nkeys, prf, out);
    return eval_host(c, packed, (size_t)nkeys * stride, compact_layout(c->depth), nkeys, prf, out);
}

int b200dpf_host_staging(b200dpf_ctx *c, int64_t nkeys, int32_t **keys_pinned)
{
    if (!c || !keys_pinned || nkeys < 1) return fail(B200DPF_EINVAL, "bad host_staging argument");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    if (c->multi) c = multi_first(c);
    const int rc = reserve_host_keys(c, (size_t)nkeys * kKeyBytes);
    if (rc) return rc;
    *keys_pinned = c->h_keys.ptr;
    return B200DPF_OK;
}

int b200dpf_eval_device(b200dpf_ctx *c, const void *keys_dev, int64_t nkeys, int prf, void *out_dev, void *cuda_stream)
{
    int rc = check_eval_args(c, keys_dev, nkeys, prf, out_dev);
    if (rc) return rc;
    if (c->multi) return fail(B200DPF_ESTATE, "multi-device contexts take host buffers (b200dpf_eval / b200dpf_eval_packed)");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    return run_eval(c, keys_dev, nkeys, prf, out_dev, reinterpret_cast<cudaStream_t>(cuda_stream));
}

int b200dpf_eval_device_acc(b200dpf_ctx *c, const void *keys_dev, int64_t nkeys, int prf, void *out_dev, void *cuda_stream)
{
    int rc = check_eval_args(c, keys_dev, nkeys, prf, out_dev);
    if (rc) return rc;
    if (c->multi) return fail(B200DPF_ESTATE, "multi-device contexts take host buffers (b200dpf_eval / b200dpf_eval_packed)");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    return run_pipeline(c, keys_dev, reference_layout(), nkeys, prf, MODE_FUSED, out_dev,
                        reinterpret_cast<cudaStream_t>(cuda_stream), false);
}

int b200dpf_expand_device(b200dpf_ctx *c, const void *keys_dev, int64_t nkeys, int prf, void *shares_dev, void *cuda_stream)
{
    int rc = check_eval_args(c, keys_dev, nkeys, prf, shares_dev);
    if (rc) return rc;
    if (c->multi) return fail(B200DPF_ESTATE, "multi-device contexts take host buffers (b200dpf_eval / b200dpf_eval_packed)");
    if (c->shard_count != 1) return fail(B200DPF_ESTATE, "expand needs an unsharded context");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    return run_pipeline(c, keys_dev, reference_layout(), nkeys, prf, MODE_EXPAND, shares_dev,
                        reinterpret_cast<cudaStream_t>(cuda_stream));
}

int64_t b200dpf_ctx_n(const b200dpf_ctx *c) { return c ? c->n : -1; }
int b200dpf_ctx_entry_size(const b200dpf_ctx *c) { return c ? c->entry_size : -1; }
int b200dpf_ctx_device(const b200dpf_ctx *c) { return c ? c->device : -1; }
int b200dpf_ctx_last_launches(const b200dpf_ctx *c)
{
    if (!c) return -1;
    return c->multi ? multi_last_launches(c) : c->last_launches;
}

int b200dpf_ctx_set_subtree_log2(b200dpf_ctx *c, int s)
{
    if (!c || s < 0 || s > 16) return fail(B200DPF_EINVAL, "subtree log2 out of range");
    c->knobs.subtree_log2 = s;
    return B200DPF_OK;
}

int b200dpf_ctx_set_option(b200dpf_ctx *c, const char *name, int value)
{
    if (!c || !name) return fail(B200DPF_EINVAL, "null argument");
    if (c->multi) return multi_set_option(c, name, value);
    struct { const char *name; int *slot; int lo, hi; } opts[] = {
        {"leaf_cache", &c->knobs.leaf_cache, 0, 1},       {"leaf_cache_mb", &c->knobs.leaf_cache_mb, 1, 1 << 20},
        {"lane_split", &c->knobs.lane_split, 0, 1},       {"frontier", &c->knobs.frontier, 0, 1},
        {"frontier_mb", &c->knobs.frontier_mb, 1, 1 << 16}, {"subtree_log2", &c->knobs.subtree_log2, 0, 16},
        {"mac_tma", &c->knobs.mac_tma, 0, 1},             {"one_launch", &c->knobs.one_launch, 0, 1},
        {"balance_top", &c->knobs.balance_top, 0, 1},     {"timing", &c->knobs.timing, 0, 1},
        {"tma_rows", &c->knobs.tma_rows, 0, 1},           {"top_log2", &c->knobs.top_log2, 0, 7},
    };
    for (auto &o : opts)
        if (std::strcmp(o.name, name) == 0) {
            if (value < o.lo || value > o.hi) return fail(B200DPF_EINVAL, "option %s=%d out of range [%d,%d]", name, value, o.lo, o.hi);
            *o.slot = value;
            return B200DPF_OK;
        }
    return fail(B200DPF_EINVAL, "unknown option '%s'", name);
}


/* ------------------------------------------------------------------------------------------- */
/* One process, several GPUs (SURVEY.md section 2.2 / 8(b): "single process drives 1/2/4/8 GPUs"). */
/* ------------------------------------------------------------------------------------------- */
}  // extern "C"

/*
 * A multi-device context owns one ordinary context per GPU and one host worker thread per GPU
 * beyond the first, so the per-device stream operations of an evaluation are issued in parallel
 * (a single thread would serialise ~10 us of launch work per device).
 *   axis ENTRIES: sub-context d is entry-range shard (d, ndev).  Every device receives every key,
 *                 evaluates its subtree, and device 0 adds the partial results with a kernel that
 *                 loads the peers' buffers over NVLink (host-side sum when peer access is absent).
 *   axis KEYS:    every sub-context holds the whole table; the batch is cut into contiguous
 *                 slices of whole key groups and nothing crosses GPUs.
 */
struct MultiState {
    int ndev = 0;
    int axis = B200DPF_AXIS_ENTRIES;
    bool peer = false;
    std::vector<b200dpf_ctx *> sub;
    std::vector<std::thread> workers;
    std::mutex m;
    std::condition_variable cv;
    std::atomic<uint64_t> gen{0};
    std::atomic<int> done{0};
    std::atomic<bool> quit{false};
    /* the job of the current generation */
    const void *keys = nullptr;
    size_t key_stride_bytes = 0;
    KeyLayout kl{};
    int64_t nkeys = 0;
    int prf = 0;
    int32_t *out = nullptr;
    bool out_pinned = false;
    std::vector<int64_t> k0, k1;      /* KEYS axis: slice of the batch per device */
    std::vector<int> rc;
    std::vector<std::string> err;

    ~MultiState()   /* the workers stop before the sub-contexts they use go */
    {
        {
            std::lock_guard<std::mutex> lk(m);
            quit.store(true, std::memory_order_release);
        }
        cv.notify_all();
        for (auto &t : workers) t.join();
        for (b200dpf_ctx *c : sub) b200dpf_destroy(c);
    }
};

b200dpf_ctx::~b200dpf_ctx()
{
    if (ev_done) cudaEventDestroy(ev_done);
    if (ev_t0) cudaEventDestroy(ev_t0);
    if (ev_t1) cudaEventDestroy(ev_t1);
    if (stream) cudaStreamDestroy(stream);
}

static inline void cpu_relax()
{
#if defined(__x86_64__) || defined(__i386__)
    __builtin_ia32_pause();
#else
    std::this_thread::yield();
#endif
}

/* Everything device d does for the current job; runs on d's own host thread with d current. */
static int multi_device_part(MultiState *M, int d)
{
    b200dpf_ctx *c = M->sub[(size_t)d];
    int64_t b = 0, e = M->nkeys;
    if (M->axis == B200DPF_AXIS_KEYS) {
        b = M->k0[(size_t)d];
        e = M->k1[(size_t)d];
        if (e <= b) return B200DPF_OK;
    }
    const int64_t nk = e - b;
    const size_t key_bytes = (size_t)nk * M->key_stride_bytes;
    const size_t out_elems = (size_t)nk * c->entry_size;
    int rc = reserve_device_io(c, key_bytes, out_elems);
    if (rc) return rc;
    rc = wait_last(c, c->stream);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_keys.ptr, static_cast<const char *>(M->keys) + (size_t)b * M->key_stride_bytes, key_bytes,
                             cudaMemcpyHostToDevice, c->stream));
    rc = run_pipeline(c, c->d_keys.ptr, M->kl, nk, M->prf, MODE_FUSED, c->d_out.ptr, c->stream);
    if (rc) return rc;
    if (M->axis == B200DPF_AXIS_KEYS) return download_out(c, M->out + (size_t)b * c->entry_size, M->out_pinned, out_elems);
    if (!M->peer) {
        rc = reserve_host_out(c, out_elems);
        if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(c->h_out.ptr, c->d_out.ptr, out_elems * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    /* ENTRIES + peer: run_pipeline recorded c->ev_done on c->stream; device 0 waits for it */
    return B200DPF_OK;
}

static void multi_worker(MultiState *M, int d)
{
    cudaSetDevice(M->sub[(size_t)d]->device);
    uint64_t seen = 0;
    for (;;) {
        int spins = 0;
        while (M->gen.load(std::memory_order_acquire) == seen && !M->quit.load(std::memory_order_acquire)) {
            if (++spins < 20000) {          /* ~1 ms of polling keeps back-to-back batches off the futex path */
                cpu_relax();
                continue;
            }
            std::unique_lock<std::mutex> lk(M->m);
            M->cv.wait(lk, [&] { return M->gen.load(std::memory_order_acquire) != seen || M->quit.load(); });
        }
        if (M->quit.load(std::memory_order_acquire)) return;
        seen = M->gen.load(std::memory_order_acquire);
        const int rc = multi_device_part(M, d);
        M->rc[(size_t)d] = rc;
        if (rc) M->err[(size_t)d] = g_err;      /* g_err is thread-local: hand the text to the caller's thread */
        M->done.fetch_add(1, std::memory_order_release);
    }
}

static b200dpf_ctx *multi_first(b200dpf_ctx *root) { return root->multi->sub[0]; }

static int multi_last_launches(const b200dpf_ctx *root)
{
    int total = 0;
    for (const b200dpf_ctx *c : root->multi->sub) total += c->last_launches;
    return total;
}

static int multi_set_option(b200dpf_ctx *root, const char *name, int value)
{
    for (b200dpf_ctx *c : root->multi->sub) {
        const int rc = b200dpf_ctx_set_option(c, name, value);
        if (rc) return rc;
    }
    return B200DPF_OK;
}

static int multi_eval_host(b200dpf_ctx *root, const void *keys, size_t key_stride_bytes, const KeyLayout &kl, int64_t nkeys,
                           int prf, int32_t *out)
{
    MultiState *M = root->multi.get();
    b200dpf_ctx *c0 = M->sub[0];
    DeviceGuard guard(c0->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c0->device);
    /* every device DMA-reads the keys from the same host buffer: it has to be pinned */
    const size_t key_bytes = (size_t)nkeys * key_stride_bytes;
    const void *src = keys;
    if (!is_pinned_host(keys)) {
        const int rc = reserve_host_keys(c0, key_bytes);
        if (rc) return rc;
        std::memcpy(c0->h_keys.ptr, keys, key_bytes);
        src = c0->h_keys.ptr;
    }
    const size_t out_elems = (size_t)nkeys * root->entry_size;
    M->keys = src;
    M->key_stride_bytes = key_stride_bytes;
    M->kl = kl;
    M->nkeys = nkeys;
    M->prf = prf;
    M->out = out;
    M->out_pinned = is_pinned_host(out);
    if (M->axis == B200DPF_AXIS_KEYS) {
        const int64_t groups = (nkeys + 31) / 32;
        const int64_t per = ((groups + M->ndev - 1) / M->ndev) * 32;
        for (int d = 0; d < M->ndev; d++) {
            M->k0[(size_t)d] = std::min<int64_t>((int64_t)d * per, nkeys);
            M->k1[(size_t)d] = std::min<int64_t>((int64_t)(d + 1) * per, nkeys);
        }
    }
    for (int d = 0; d < M->ndev; d++) M->rc[(size_t)d] = B200DPF_OK;
    M->done.store(0, std::memory_order_relaxed);
    {
        std::lock_guard<std::mutex> lk(M->m);
        M->gen.fetch_add(1, std::memory_order_release);
    }
    M->cv.notify_all();
    M->rc[0] = multi_device_part(M, 0);
    if (M->rc[0]) M->err[0] = g_err;
    while (M->done.load(std::memory_order_acquire) < M->ndev - 1) cpu_relax();
    for (int d = 0; d < M->ndev; d++)
        if (M->rc[(size_t)d]) return fail(M->rc[(size_t)d], "device %d: %s", M->sub[(size_t)d]->device, M->err[(size_t)d].c_str());
    if (M->axis == B200DPF_AXIS_KEYS) return B200DPF_OK;     /* every device delivered its own rows */

    if (M->peer) {
        /* device 0: wait for every shard's kernel, then add the peers' partials over NVLink */
        PeerParts parts;
        parts.n = 0;
        for (int d = 1; d < M->ndev; d++) {
            CUDA_TRY(cudaStreamWaitEvent(c0->stream, M->sub[(size_t)d]->ev_done, 0));
            parts.p[parts.n++] = reinterpret_cast<const uint32_t *>(M->sub[(size_t)d]->d_out.ptr);
        }
        CUDA_TRY(launch_sum_partials(reinterpret_cast<uint32_t *>(c0->d_out.ptr), parts, out_elems, c0->sm_count, c0->stream));
        return download_out(c0, out, M->out_pinned, out_elems);
    }
    /* no peer access between these devices: every shard already copied its partial to pinned
     * host memory; wrapping 32-bit adds on the host */
    uint32_t *o = reinterpret_cast<uint32_t *>(out);
    std::memcpy(o, c0->h_out.ptr, out_elems * sizeof(int32_t));
    for (int d = 1; d < M->ndev; d++) {
        const uint32_t *part = reinterpret_cast<const uint32_t *>(M->sub[(size_t)d]->h_out.ptr);
        for (size_t i = 0; i < out_elems; i++) o[i] += part[i];
    }
    return B200DPF_OK;
}

extern "C" {

int b200dpf_create_multi(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, const int *devices, int ndev,
                         int axis)
{
    if (!out) return fail(B200DPF_EINVAL, "null ctx out pointer");
    *out = nullptr;
    if (!devices || ndev < 1 || ndev > 16) return fail(B200DPF_EINVAL, "need 1..16 devices (got %d)", ndev);
    if (axis != B200DPF_AXIS_AUTO && axis != B200DPF_AXIS_ENTRIES && axis != B200DPF_AXIS_KEYS)
        return fail(B200DPF_EINVAL, "unknown axis %d", axis);
    for (int i = 0; i < ndev; i++)
        for (int j = 0; j < i; j++)
            if (devices[i] == devices[j]) return fail(B200DPF_EINVAL, "device %d listed twice", devices[i]);
    const bool pow2 = (ndev & (ndev - 1)) == 0;
    if (axis == B200DPF_AXIS_AUTO)
        axis = (pow2 && n > B200DPF_AUTO_KEYS_MAX_N && (int64_t)ndev <= n / 2) ? B200DPF_AXIS_ENTRIES : B200DPF_AXIS_KEYS;
    if (axis == B200DPF_AXIS_ENTRIES && (!pow2 || (int64_t)ndev > n / 2))
        return fail(B200DPF_EINVAL, "entry-range sharding needs a power-of-two device count <= n/2 (got %d)", ndev);

    std::unique_ptr<b200dpf_ctx> root(new (std::nothrow) b200dpf_ctx());
    if (root) root->multi.reset(new (std::nothrow) MultiState());
    if (!root || !root->multi) return fail(B200DPF_ENOMEM, "out of host memory");
    MultiState *M = root->multi.get();
    root->n = n;
    root->depth = ilog2(n);
    root->entry_size = entry_size;
    root->device = devices[0];
    M->ndev = ndev;
    M->axis = axis;
    M->k0.assign((size_t)ndev, 0);
    M->k1.assign((size_t)ndev, 0);
    M->rc.assign((size_t)ndev, 0);
    M->err.assign((size_t)ndev, std::string());
    for (int d = 0; d < ndev; d++) {
        b200dpf_ctx *c = nullptr;
        const int rc = axis == B200DPF_AXIS_ENTRIES ? b200dpf_create(&c, table, n, entry_size, devices[d], d, ndev)
                                                    : b200dpf_create(&c, table, n, entry_size, devices[d], 0, 1);
        if (rc) return rc;     /* message already set by b200dpf_create; the root destroys the sub-contexts made */
        M->sub.push_back(c);
    }
    /* device 0 reads the other shards' partial results in place: NVLink peer mappings */
    M->peer = axis == B200DPF_AXIS_ENTRIES && ndev > 1;
    if (M->peer) {
        DeviceGuard guard(devices[0]);
        for (int d = 1; d < ndev && M->peer; d++) {
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, devices[0], devices[d]) != cudaSuccess || !can) M->peer = false;
        }
        for (int d = 1; d < ndev && M->peer; d++) {
            const cudaError_t e = cudaDeviceEnablePeerAccess(devices[d], 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) M->peer = false;
        }
        cudaGetLastError();
    }
    for (int d = 1; d < ndev; d++) M->workers.emplace_back(multi_worker, M, d);
    *out = root.release();
    return B200DPF_OK;
}

/* ------------------------------------------------------------------------------------------- */
/* Grouped evaluation: the batch-PIR front end (SURVEY.md section 8(f) rank 4).                  */
/* ------------------------------------------------------------------------------------------- */
int b200dpf_group_create(b200dpf_ctx **out, const int32_t *const *tables, const int64_t *n, int nbins, int entry_size,
                         int device)
{
    if (!out) return fail(B200DPF_EINVAL, "null ctx out pointer");
    *out = nullptr;
    if (!tables || !n || nbins < 1 || nbins > (1 << 20)) return fail(B200DPF_EINVAL, "bad bin list (nbins=%d)", nbins);
    if (entry_size < 1 || entry_size > 4096) return fail(B200DPF_EINVAL, "entry_size=%d out of range [1,4096]", entry_size);
    int64_t n_max = 0, rows = 0;
    for (int g = 0; g < nbins; g++) {
        if (!tables[g]) return fail(B200DPF_EINVAL, "bin %d: null table", g);
        if (n[g] < 2 || n[g] > ((int64_t)1 << 31) || (n[g] & (n[g] - 1)) != 0)
            return fail(B200DPF_EINVAL, "bin %d: size n=%lld must be a power of two in [2, 2^31]", g, (long long)n[g]);
        n_max = std::max(n_max, n[g]);
        rows += n[g];
    }
    std::optional<DeviceGuard> guard;
    std::unique_ptr<b200dpf_ctx> c;
    int rc = ctx_open(device, false, &guard, &c);     /* grouped contexts keep the default knobs */
    if (rc) return rc;
    c->bins.reset(new (std::nothrow) GroupBins());
    if (!c->bins) return fail(B200DPF_ENOMEM, "out of host memory");
    GroupBins *B = c->bins.get();
    c->n = n_max;                      /* the launch plan (shared memory for correction words) is sized by the deepest bin */
    c->depth = ilog2(n_max);
    c->entry_size = entry_size;
    c->entry_pad = (entry_size + 15) & ~15;       /* 16 columns per pass */
    c->n_local = n_max;
    c->depth_local = c->depth;
    CUDA_TRY(cudaMemsetAsync(c->d_gridbar.ptr, 0, sizeof(uint32_t), c->stream));
    if (!c->coop_ok) return fail(B200DPF_ECUDA, "grouped evaluation needs cooperative launch support");
    const size_t table_bytes = (size_t)rows * (size_t)c->entry_pad * sizeof(int32_t);
    rc = c->d_table.reserve(table_bytes);
    if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_table.ptr, 0, table_bytes, c->stream));
    DeviceBuffer<int32_t> d_stage;
    rc = d_stage.reserve((size_t)n_max * entry_size * sizeof(int32_t));
    if (rc) return rc;
    uint64_t row0 = 0;
    for (int g = 0; g < nbins; g++) {
        /* each bin in its own breadth-first leaf order (bit reversal over ITS depth), 64-byte rows */
        const int depth = ilog2(n[g]);
        B->n.push_back(n[g]);
        B->depth.push_back(depth);
        B->row_off.push_back(row0);
        CUDA_TRY(cudaMemcpyAsync(d_stage.ptr, tables[g], (size_t)n[g] * entry_size * sizeof(int32_t), cudaMemcpyDefault, c->stream));
        CUDA_TRY(launch_permute_table(d_stage.ptr, c->d_table.ptr + row0 * (uint64_t)c->entry_pad, (uint64_t)n[g], depth,
                                      entry_size, c->entry_pad, c->sm_count, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));    /* the staging buffer is reused */
        row0 += (uint64_t)n[g];
    }
    *out = c.release();
    return B200DPF_OK;
}

int b200dpf_group_eval(b200dpf_ctx *c, const int32_t *keys, const int32_t *bins, int64_t nkeys, int prf, int32_t *out)
{
    if (!c || !c->bins) return fail(B200DPF_ESTATE, "not a grouped context (b200dpf_group_create)");
    if (!keys || !bins || !out) return fail(B200DPF_EINVAL, "null buffer");
    if (nkeys < 1 || nkeys > (int64_t)1 << 24) return fail(B200DPF_EINVAL, "nkeys=%lld out of range", (long long)nkeys);
    if (prf < B200DPF_PRF_DUMMY || prf > B200DPF_PRF_AES128) return fail(B200DPF_EINVAL, "unknown prf id %d", prf);
    GroupBins *B = c->bins.get();
    const int nbins = (int)B->n.size();
    /* counting sort by bin: a key group must not mix bins */
    std::vector<int64_t> count((size_t)nbins + 1, 0);
    for (int64_t b = 0; b < nkeys; b++) {
        const int g = bins[b];
        if (g < 0 || g >= nbins) return fail(B200DPF_EINVAL, "key %lld: bin %d out of range [0,%d)", (long long)b, g, nbins);
        if (host::key_n(keys + b * host::KEY_WORDS) != B->n[(size_t)g])
            return fail(B200DPF_EINVAL, "key %lld was generated for n=%lld, bin %d has n=%lld", (long long)b,
                        (long long)host::key_n(keys + b * host::KEY_WORDS), g, (long long)B->n[(size_t)g]);
        count[(size_t)g + 1]++;
    }
    for (int g = 0; g < nbins; g++) count[(size_t)g + 1] += count[(size_t)g];
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    /* keys travel in the compact layout, one stride for all bins (that of the deepest): a key for a
     * 2^10-entry bin has 672 live bytes of its 2096 */
    const KeyLayout kl = compact_layout(c->depth);
    const size_t stride = (size_t)kl.stride_v * 16u;
    const size_t key_bytes = (size_t)nkeys * stride;
    int rc = reserve_host_keys(c, key_bytes);
    if (rc) return rc;
    B->perm.assign((size_t)nkeys, 0);
    {
        std::vector<int64_t> next(count.begin(), count.end() - 1);
        for (int64_t b = 0; b < nkeys; b++) B->perm[(size_t)(next[(size_t)bins[b]]++)] = b;
        uint8_t *stage = reinterpret_cast<uint8_t *>(c->h_keys.ptr);
        auto pack_range = [&](int64_t p0, int64_t p1) {
            for (int64_t pos = p0; pos < p1; pos++) {
                const int64_t b = B->perm[(size_t)pos];
                pack_compact(keys + b * host::KEY_WORDS, stage + (size_t)pos * stride, B->depth[(size_t)bins[b]]);
            }
        };
        const int nthr = (int)std::min<int64_t>(std::min<int64_t>(8, std::max(1u, std::thread::hardware_concurrency())), nkeys / 2048 + 1);
        std::vector<std::thread> pool;
        for (int t = 1; t < nthr; t++) pool.emplace_back(pack_range, nkeys * t / nthr, nkeys * (t + 1) / nthr);
        pack_range(0, nkeys / nthr);
        for (auto &th : pool) th.join();
    }
    /* key groups and their work-item size: big items amortise the root-to-subtree walk every item
     * pays (there is no frontier: bins are small), small items keep every warp busy */
    SmemLayout L;
    rc = smem_layout(c, prf, 4, MODE_GROUPED, &L);
    if (rc) return rc;
    const int64_t warps = (int64_t)L.grid * (L.threads / 32);
    int64_t ngroups = 0;
    for (int g = 0; g < nbins; g++) ngroups += (count[(size_t)g + 1] - count[(size_t)g] + 31) / 32;
    int s_target = c->knobs.subtree_log2 > 0 ? c->knobs.subtree_log2 : 6;
    s_target = std::min(s_target, L.s_max);
    if (c->knobs.subtree_log2 <= 0) {
        for (; s_target > 3; s_target--) {
            int64_t items = 0;
            for (int g = 0; g < nbins; g++) {
                const int64_t kg = (count[(size_t)g + 1] - count[(size_t)g] + 31) / 32;
                items += kg << std::max(0, B->depth[(size_t)g] - s_target);
            }
            if (items >= 2 * warps) break;
        }
    }
    const size_t descs_bytes = std::max<size_t>((size_t)ngroups, 1024) * sizeof(GroupDesc);
    rc = B->h_descs.reserve(descs_bytes);
    if (!rc) rc = B->d_descs.reserve(descs_bytes);
    if (rc) return rc;
    int s_max = 1;
    {
        int64_t gi = 0;
        for (int g = 0; g < nbins; g++) {
            const int depth = B->depth[(size_t)g];
            const int s = std::max(1, std::min(depth, s_target));
            for (int64_t k = count[(size_t)g]; k < count[(size_t)g + 1]; k += 32, gi++) {
                GroupDesc &d = B->h_descs.ptr[gi];
                d.key_first = (uint32_t)k;
                d.nkeys = (uint32_t)std::min<int64_t>(32, count[(size_t)g + 1] - k);
                d.depth = depth;
                d.s = s;
                d.nsub = (uint32_t)1 << (depth - s);
                d.pad = 0;
                d.table_off_v = B->row_off[(size_t)g] * (uint64_t)(c->entry_pad / 4);
                s_max = std::max(s_max, s);
            }
        }
    }
    const int passes = c->entry_pad / 16;
    const size_t out_elems = (size_t)nkeys * c->entry_size;
    rc = reserve_device_io(c, key_bytes, out_elems);
    if (!rc) rc = reserve_host_out(c, out_elems);
    if (rc) return rc;
    const size_t n_counters = (size_t)passes * (size_t)ngroups;
    rc = c->d_counters.reserve(n_counters * sizeof(uint32_t));
    if (!rc) rc = wait_last(c, c->stream);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_keys.ptr, c->h_keys.ptr, key_bytes, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaMemcpyAsync(B->d_descs.ptr, B->h_descs.ptr, (size_t)ngroups * sizeof(GroupDesc), cudaMemcpyHostToDevice, c->stream));
    if (c->coop_state_dirty) {
        CUDA_TRY(cudaMemsetAsync(c->d_gridbar.ptr, 0, sizeof(uint32_t), c->stream));
        c->bar_epoch = 0;
        c->coop_state_dirty = false;
    }
    EvalParams p;
    size_t smem;
    fill_common(c, L, s_max, nkeys, 5, &p, &smem);
    p.key_groups = (int)ngroups;
    p.keys = reinterpret_cast<const uint4 *>(c->d_keys.ptr);
    p.key_stride_v = kl.stride_v; p.key_root_v = kl.root_v; p.key_compact = kl.compact;
    p.groups = B->d_descs.ptr;
    fill_phase(L, s_max, &p.main);
    p.main.counters = c->d_counters.ptr;
    p.out = reinterpret_cast<uint32_t *>(c->d_out.ptr);
    /* one cooperative launch per 16 columns; the first one clears the result and every pass's tickets */
    p.fuse_top = 1;
    p.zero_a = p.out;
    p.zero_a_words = out_elems;
    p.zero_b = c->d_counters.ptr;
    p.zero_b_words = n_counters;
    c->last_launches = 0;
    CUDA_TRY(cudaEventRecord(c->ev_t0, c->stream));
    for (int pass = 0; pass < passes; pass++) {
        p.col_off_v = (uint32_t)(pass * 4);
        p.col_off = (uint32_t)(pass * 16);
        p.ncols = (uint32_t)std::max(0, std::min(16, c->entry_size - pass * 16));
        if (p.ncols == 0) break;
        p.main.counters = c->d_counters.ptr + (size_t)pass * (size_t)ngroups;
        if (p.fuse_top) {
            p.grid_bar = c->d_gridbar.ptr;
            c->bar_epoch += (uint32_t)L.grid;
            p.grid_bar_target = c->bar_epoch;
        }
        const cudaError_t e = launch_eval(prf, 4, MODE_GROUPED, p, L.grid, smem, c->stream);
        if (e != cudaSuccess) {
            c->coop_state_dirty = true;
            return fail(B200DPF_ECUDA, "grouped evaluation launch: %s", cudaGetErrorString(e));
        }
        c->last_launches++;
        p.fuse_top = 0;
    }
    CUDA_TRY(cudaEventRecord(c->ev_t1, c->stream));
    c->timed = true;
    CUDA_TRY(cudaMemcpyAsync(c->h_out.ptr, c->d_out.ptr, out_elems * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    rc = mark_last(c, c->stream);
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (int64_t pos = 0; pos < nkeys; pos++)       /* back to the caller's order */
        std::memcpy(out + B->perm[(size_t)pos] * c->entry_size, c->h_out.ptr + pos * c->entry_size, sizeof(int32_t) * (size_t)c->entry_size);
    return B200DPF_OK;
}

/* ------------------------------------------------------------------------------------------- */
/* Row updates of a live table.                                                                  */
/* ------------------------------------------------------------------------------------------- */
}  // extern "C"

namespace {

constexpr int64_t kMaxUpdateCount = 0x7fffffff;   /* occurrence numbers are 32-bit, as is the sort's item count */

/* Update scratch (one allocation, every section 256-byte aligned):
 *   [idx int64 | bins int32 | rows int32 [count][entry_size]]   host paths only: the caller's rows copied in
 *   pos_in | pos_out | ord_in | ord_out                          uint32 [count] each
 *   sort temporary                                               cub::DeviceRadixSort::SortPairs */
struct UpdateLayout {
    size_t off_idx, off_bins, off_rows, off_work[4], off_temp, temp_bytes, total;
    int end_bit;
};

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

/* rows of the device table; also the skip marker of the update kernels (larger than every position) */
uint64_t update_table_rows(const b200dpf_ctx *c)
{
    return c->bins ? c->bins->row_off.back() + (uint64_t)c->bins->n.back() : (uint64_t)c->n_local;
}

/* Grow the scratch for `count` rows (staged: the inputs are copied into it) and order everything that
 * follows on `stream` after the context's previous evaluation or update: the update writes the table
 * those read, and the scratch is the previous update's. */
int update_begin(b200dpf_ctx *c, int64_t count, bool staged, bool with_bins, cudaStream_t stream, UpdateLayout *L)
{
    const uint64_t rows = update_table_rows(c);
    if (rows >= 0xffffffffull) return fail(B200DPF_EINVAL, "table of %llu rows too large for row updates", (unsigned long long)rows);
    L->end_bit = 1;
    while (L->end_bit < 32 && (rows >> L->end_bit) != 0) L->end_bit++;
    CUDA_TRY(update_temp_bytes(count, L->end_bit, &L->temp_bytes));
    size_t off = 0;
    L->off_idx = off;
    if (staged) off = align256(off + (size_t)count * sizeof(int64_t));
    L->off_bins = off;
    if (staged && with_bins) off = align256(off + (size_t)count * sizeof(int32_t));
    L->off_rows = off;
    if (staged) off = align256(off + (size_t)count * (size_t)c->entry_size * sizeof(int32_t));
    for (int k = 0; k < 4; k++) {
        L->off_work[k] = off;
        off = align256(off + (size_t)count * sizeof(uint32_t));
    }
    L->off_temp = off;
    L->total = align256(off + L->temp_bytes);
    const int rc = c->d_update.reserve(L->total);
    return rc ? rc : wait_last(c, stream);
}

/* Enqueue the scatter (inputs in device memory) and record it as the context's last operation. */
int update_run(b200dpf_ctx *c, const UpdateLayout &L, const int64_t *idx, const int32_t *bins, const int32_t *rows,
               int64_t count, cudaStream_t stream)
{
    char *s = c->d_update.ptr;
    UpdateParams u;
    std::memset(&u, 0, sizeof u);
    u.idx = idx;
    u.bins = bins;
    if (bins) {
        u.bin_info = c->bins->d_bin_info.ptr;
        u.nbins = (int)c->bins->n.size();
    }
    u.rows = rows;
    u.count = count;
    u.n = c->n;
    u.own_mask = (uint32_t)c->shard_count - 1u;
    u.own_val = bitrev_host((uint32_t)c->shard_rank, c->shard_bits);
    u.shift = c->shard_bits;
    u.depth = c->depth_local;
    u.table_rows = (uint32_t)update_table_rows(c);
    u.lane_bits = c->lane_bits;
    u.table = c->d_table.ptr;
    u.cols = c->entry_size;
    u.stride = c->entry_pad;
    UpdateWork w;
    w.pos_in = reinterpret_cast<uint32_t *>(s + L.off_work[0]);
    w.pos_out = reinterpret_cast<uint32_t *>(s + L.off_work[1]);
    w.ord_in = reinterpret_cast<uint32_t *>(s + L.off_work[2]);
    w.ord_out = reinterpret_cast<uint32_t *>(s + L.off_work[3]);
    w.temp = s + L.off_temp;
    w.temp_bytes = L.temp_bytes;
    CUDA_TRY(launch_update_rows(u, w, L.end_bit, c->sm_count, stream));
    return mark_last(c, stream);
}

/* Host path on one single-device context (device already current, inputs validated): copy the rows this
 * context owns into the scratch and enqueue the scatter on the context's stream.  The caller synchronises. */
int update_host_enqueue(b200dpf_ctx *c, const int64_t *idx, const int32_t *bins, const int32_t *rows, int64_t count)
{
    std::vector<int64_t> own_idx;
    std::vector<int32_t> own_rows;
    if (c->shard_count > 1) {             /* a shard copies only its own rows */
        const uint32_t mask = (uint32_t)c->shard_count - 1u, val = bitrev_host((uint32_t)c->shard_rank, c->shard_bits);
        for (int64_t j = 0; j < count; j++)
            if (((uint32_t)(idx[j] >> c->lane_bits) & mask) == val) {
                own_idx.push_back(idx[j]);
                own_rows.insert(own_rows.end(), rows + j * c->entry_size, rows + (j + 1) * c->entry_size);
            }
        idx = own_idx.data();
        rows = own_rows.data();
        count = (int64_t)own_idx.size();
    }
    if (count == 0) return B200DPF_OK;
    UpdateLayout L;
    int rc = update_begin(c, count, true, bins != nullptr, c->stream, &L);
    if (rc) return rc;
    char *s = c->d_update.ptr;
    CUDA_TRY(cudaMemcpyAsync(s + L.off_idx, idx, (size_t)count * sizeof(int64_t), cudaMemcpyHostToDevice, c->stream));
    if (bins) CUDA_TRY(cudaMemcpyAsync(s + L.off_bins, bins, (size_t)count * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaMemcpyAsync(s + L.off_rows, rows, (size_t)count * (size_t)c->entry_size * sizeof(int32_t),
                             cudaMemcpyHostToDevice, c->stream));
    return update_run(c, L, reinterpret_cast<const int64_t *>(s + L.off_idx),
                      bins ? reinterpret_cast<const int32_t *>(s + L.off_bins) : nullptr,
                      reinterpret_cast<const int32_t *>(s + L.off_rows), count, c->stream);
}

int check_update_args(const b200dpf_ctx *c, const void *idx, const void *rows, int64_t count)
{
    if (!c) return fail(B200DPF_EINVAL, "null context");
    if (count < 0 || count > kMaxUpdateCount) return fail(B200DPF_EINVAL, "update count=%lld out of range [0, 2^31)", (long long)count);
    if (count > 0 && (!idx || !rows)) return fail(B200DPF_EINVAL, "null buffer");
    return B200DPF_OK;
}

}  // namespace

extern "C" {

int b200dpf_update_rows(b200dpf_ctx *c, const int64_t *indices, const int32_t *rows, int64_t count)
{
    int rc = check_update_args(c, indices, rows, count);
    if (rc) return rc;
    if (c->bins) return fail(B200DPF_ESTATE, "grouped context: use b200dpf_group_update_rows");
    if (!c->d_table.ptr && !c->multi) return fail(B200DPF_ESTATE, "context has no table");
    for (int64_t j = 0; j < count; j++)
        if (indices[j] < 0 || indices[j] >= c->n)
            return fail(B200DPF_EINVAL, "update %lld: index %lld out of range [0, %lld)", (long long)j, (long long)indices[j],
                        (long long)c->n);
    if (count == 0) return B200DPF_OK;
    std::vector<b200dpf_ctx *> subs = c->multi ? c->multi->sub : std::vector<b200dpf_ctx *>{c};
    /* every device's copies and kernels are issued before the first synchronisation */
    for (b200dpf_ctx *s : subs) {
        DeviceGuard guard(s->device);
        if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", s->device);
        rc = update_host_enqueue(s, indices, nullptr, rows, count);
        if (rc) return rc;
    }
    for (b200dpf_ctx *s : subs) {
        DeviceGuard guard(s->device);
        CUDA_TRY(cudaStreamSynchronize(s->stream));
    }
    return B200DPF_OK;
}

int b200dpf_update_rows_device(b200dpf_ctx *c, const int64_t *indices_dev, const int32_t *rows_dev, int64_t count,
                               void *cuda_stream)
{
    int rc = check_update_args(c, indices_dev, rows_dev, count);
    if (rc) return rc;
    if (c->multi) return fail(B200DPF_EINVAL, "multi-device contexts take host buffers (b200dpf_update_rows)");
    if (c->bins) return fail(B200DPF_ESTATE, "grouped context: use b200dpf_group_update_rows");
    if (!c->d_table.ptr) return fail(B200DPF_ESTATE, "context has no table");
    if (count == 0) return B200DPF_OK;
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    const cudaStream_t stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    UpdateLayout L;
    rc = update_begin(c, count, false, false, stream, &L);
    if (rc) return rc;
    return update_run(c, L, indices_dev, nullptr, rows_dev, count, stream);
}

int b200dpf_group_update_rows(b200dpf_ctx *c, const int32_t *bins, const int64_t *indices, const int32_t *rows, int64_t count)
{
    int rc = check_update_args(c, indices, rows, count);
    if (rc) return rc;
    if (!c->bins) return fail(B200DPF_ESTATE, "not a grouped context (b200dpf_group_create)");
    if (count > 0 && !bins) return fail(B200DPF_EINVAL, "null buffer");
    GroupBins *B = c->bins.get();
    const int nbins = (int)B->n.size();
    for (int64_t j = 0; j < count; j++) {
        if (bins[j] < 0 || bins[j] >= nbins)
            return fail(B200DPF_EINVAL, "update %lld: bin %d out of range [0,%d)", (long long)j, bins[j], nbins);
        if (indices[j] < 0 || indices[j] >= B->n[(size_t)bins[j]])
            return fail(B200DPF_EINVAL, "update %lld: index %lld out of range [0, %lld) of bin %d", (long long)j,
                        (long long)indices[j], (long long)B->n[(size_t)bins[j]], bins[j]);
    }
    if (count == 0) return B200DPF_OK;
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    if (!B->d_bin_info.ptr) {
        std::vector<uint2> info((size_t)nbins);
        for (int g = 0; g < nbins; g++) info[(size_t)g] = make_uint2((uint32_t)B->row_off[(size_t)g], (uint32_t)B->depth[(size_t)g]);
        rc = B->d_bin_info.reserve(info.size() * sizeof(uint2));
        if (rc) return rc;
        CUDA_TRY(cudaMemcpy(B->d_bin_info.ptr, info.data(), info.size() * sizeof(uint2), cudaMemcpyHostToDevice));
    }
    rc = update_host_enqueue(c, indices, bins, rows, count);
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    return B200DPF_OK;
}

double b200dpf_ctx_last_device_ms(b200dpf_ctx *c)
{
    if (!c) return -1.0;
    if (c->multi) c = multi_first(c);
    if (!c->timed) return -1.0;
    DeviceGuard guard(c->device);
    float ms = -1.0f;
    if (cudaEventSynchronize(c->ev_t1) != cudaSuccess || cudaEventElapsedTime(&ms, c->ev_t0, c->ev_t1) != cudaSuccess) {
        cudaGetLastError();
        return -1.0;
    }
    return (double)ms;
}

int b200dpf_group_bins(const b200dpf_ctx *c) { return (c && c->bins) ? (int)c->bins->n.size() : 0; }


int b200dpf_ctx_read_timing(b200dpf_ctx *c, uint64_t *stamps, int max_blocks, int *nblocks)
{
    if (!c || !stamps || !nblocks) return fail(B200DPF_EINVAL, "null argument");
    if (c->multi) c = multi_first(c);
    *nblocks = 0;
    if (!c->d_timing.ptr) return B200DPF_OK;
    DeviceGuard guard(c->device);
    const int nb = std::min(max_blocks, (int)(c->d_timing.cap / (8 * sizeof(unsigned long long))));
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(stamps, c->d_timing.ptr, (size_t)nb * 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    *nblocks = nb;
    return B200DPF_OK;
}

int b200dpf_ctx_device_count(const b200dpf_ctx *c) { return !c ? -1 : (c->multi ? c->multi->ndev : 1); }

int b200dpf_ctx_axis(const b200dpf_ctx *c)
{
    if (!c) return -1;
    if (c->multi) return c->multi->axis;
    return c->shard_count > 1 ? B200DPF_AXIS_ENTRIES : B200DPF_AXIS_AUTO;
}

}  // extern "C"
