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

/* The shape of one table or bin, made by table_shape.  Its keys are made for 2^(depth + lane_bits) rows. */
struct TableShape {
    int64_t n;          /* live rows */
    int depth;          /* leaf levels of the key tree */
    int64_t rows;       /* rows of the device table, padding included */
    int room;           /* log2 leaves of the largest work item inside those rows: depth, or less if trimmed */
    uint64_t first;     /* first device row */
};

}  // namespace

struct SmemLayoutCache;   /* per (prf, nv, mode) launch layouts, filled on first use */
struct MultiState;        /* b200dpf_create_multi: per-device sub-contexts + worker threads */
struct GroupBins;         /* b200dpf_group_create: many tables ("bins") behind one context */

struct b200dpf_ctx {
    std::unique_ptr<MultiState> multi;   /* non-null: this context only fans out to multi->sub[] */
    std::unique_ptr<GroupBins> bins;     /* non-null: grouped (batch-PIR) context, use b200dpf_group_eval */
    std::unique_ptr<SmemLayoutCache> layouts;
    int device = 0;
    TableShape shape{};      /* the whole table's; grouped: the largest bin's n, the deepest bin's depth, all bins' rows */
    int entry_size = 0;
    int entry_pad = 0;       /* row length in int32: 16, 32 or a multiple of 64     */
    int shard_rank = 0, shard_count = 1, shard_bits = 0;
    /* this shard's part of the table: the tree below the shard root and the rows of d_table */
    int depth_local() const { return shape.depth - shard_bits; }
    int64_t rows_local() const { return shape.rows >> shard_bits; }
    /* the kind of key the context takes (host::KindInfo): standard, early-terminated (b200dpf_create_et) or
     * XOR-shared (b200dpf_create_xor).  A leaf carries 2^lane_bits() table rows: the shape's n and rows, the
     * table, the leaf cache and the results count rows; depths, the shards, the work items and the frontier
     * count leaves. */
    int kind = host::KIND_STANDARD;
    int lane_bits() const { return host::kKinds[kind].lane_bits; }
    /* trimmed (b200dpf_create_trimmed, b200dpf_group_create_trimmed): row r is device row r, at leaf position
     * r >> lane_bits of a tree over trimmed_domain(n) rows (table_shape) */
    bool trimmed = false;
    RowPlacement place{};             /* where this table's (or shard's) rows live in d_table; not used when grouped */
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
    /* tuning knobs, described by kKnobs: defaults from the environment, read ONCE at b200dpf_create;
     * changed per context with b200dpf_ctx_set_option */
    struct Knobs {
        int leaf_cache, leaf_cache_mb, lane_split, frontier, frontier_mb, subtree_log2, mac_tma, one_launch,
            balance_top, timing, top_log2, tma_rows;
        Knobs();   /* the defaults of kKnobs */
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

/* One tuning option: its field, default, environment variable (read by b200dpf_create and the other
 * plain-context constructors; unchecked, as atoi reads it) and b200dpf_ctx_set_option name and range. */
using Kn = b200dpf_ctx::Knobs;
using KnobField = int Kn::*;
struct KnobInfo { KnobField field; int dflt; const char *env, *name; int lo, hi; };
constexpr KnobInfo kKnobs[] = {
    {&Kn::leaf_cache, 1, "B200DPF_LEAF_CACHE", "leaf_cache", 0, 1},                /* wide entries: cache leaves, MAC-only passes */
    {&Kn::leaf_cache_mb, 16384, "B200DPF_LEAF_CACHE_MB", "leaf_cache_mb", 1, 1 << 20},  /* cap; larger batches go in chunks */
    {&Kn::lane_split, 1, "B200DPF_LANE_SPLIT", "lane_split", 0, 1},                /* batches < 32 keys: lane = (key, subtree) */
    {&Kn::frontier, 1, "B200DPF_FRONTIER", "frontier", 0, 1},                      /* expand the tree top once per evaluation */
    {&Kn::frontier_mb, 256, "B200DPF_FRONTIER_MB", "frontier_mb", 1, 1 << 16},
    {&Kn::subtree_log2, 0, "B200DPF_S", "subtree_log2", 0, 16},                    /* 0 = automatic */
    {&Kn::mac_tma, 1, "B200DPF_MAC_TMA", "mac_tma", 0, 1},                         /* cp.async.bulk-staged MAC passes */
    {&Kn::one_launch, 1, "B200DPF_ONE_LAUNCH", "one_launch", 0, 1},                /* whole evaluation as one cooperative launch */
    {&Kn::balance_top, 1, "B200DPF_BALANCE_TOP", "balance_top", 0, 1},             /* even per-block shares of the tree-top phase */
    {&Kn::timing, 0, "B200DPF_TIMING", "timing", 0, 1},                            /* per-block phase time stamps (diagnostics) */
    {&Kn::top_log2, 0, "B200DPF_TOP_LOG2", "top_log2", 0, 7},   /* log2 leaves-of-the-frontier per tree-top item (0 = estimate) */
    /* fused kernel: stage each item's rows with cp.async.bulk (16-column tables, Salsa/ChaCha/dummy); on an H100 at
     * n=2^20 +4 % for Salsa20, -2 % for ChaCha20 against broadcast loads, other sizes unmeasured -- so off */
    {&Kn::tma_rows, 0, "B200DPF_TMA_ROWS", "tma_rows", 0, 1},
};

}  // namespace

b200dpf_ctx::Knobs::Knobs() { for (const KnobInfo &k : kKnobs) this->*k.field = k.dflt; }

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
    const BlockShape shape = eval_block_shape(prf, nv, mode);
    L->threads = shape.threads;
    L->blocks_per_sm = shape.min_blocks;
    L->grid = c->sm_count * L->blocks_per_sm;
    int max_smem = 0;
    CUDA_TRY(eval_max_smem(prf, nv, mode, &max_smem));
    int sm_total = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&sm_total, cudaDevAttrMaxSharedMemoryPerMultiprocessor, c->device));
    /* every resident block also pays the 1 KiB system reservation */
    int budget = std::min(max_smem, sm_total / L->blocks_per_sm - 1024);
    budget &= ~15;
    L->budget = budget;

    L->meta_cw = (uint32_t)c->shape.depth * 4u * 32u * 16u;
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
        else return fail(B200DPF_EINVAL, "depth %d needs more shared memory than available", c->shape.depth);
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
        if ((int64_t)budget < (int64_t)L->off_lo) return fail(B200DPF_EINVAL, "depth %d needs more shared memory than available", c->shape.depth);
        L->cap_lo = (int)(((uint32_t)budget - L->off_lo) / L->level_bytes);
        L->off_hi = L->off_lo;
        L->cap_hi = 0;
        L->smem_fixed = 0;
    }
    L->s_max = 1 + L->cap_lo + L->cap_hi;
    return B200DPF_OK;
}

/* Dynamic shared memory of a launch on layout L whose deepest pending-sibling stack is s levels */
size_t smem_bytes(const SmemLayout &L, int s)
{
    return L.smem_fixed ? L.smem_fixed : (size_t)L.off_lo + (size_t)(s > 1 ? s - 1 : 0) * L.level_bytes;
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

/* compact form of one key straight into `dst` (b200dpf_key_pack without the checks); `magic` is its kind's */
inline void pack_compact(const int32_t *key, uint8_t *dst, int depth, const char *magic)
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

/* What the contexts and the launch planner do differently per kind of key (host::kKinds has the key
 * format): the kernel modes, and the limits of one kind. */
struct KindOps {
    int mode_fused, mode_expand;
    int mode_grouped;
    int mode_grouped_dev;   /* the grouped mode of lists planned on the device (b200dpf_group_eval_device_bins) */
    int max_nv;             /* fused passes: at most 4 * max_nv columns (early-terminated 32, XOR-shared 16) */
    bool leaf_cache;        /* wide entries may cache leaves (XOR-shared: a further 16 columns re-walk the tree) */
    bool tma_rows;          /* the B200DPF_TMA_ROWS variant exists */
    int min_kpw_log2;       /* fused launches: at least 2^this keys per warp (the XOR kernel splits rows across a
                             * key quad; the missing keys of a smaller batch are duplicates whose results are dropped) */
    int leaf_items;         /* > 0: automatic s for leaves of many rows -- items down to s = 1, this many per warp */
    const char *gen;        /* the generator of the kind's keys, in messages */
};
constexpr KindOps kKindOps[host::KIND_COUNT] = {
    {MODE_FUSED, MODE_EXPAND, MODE_GROUPED, MODE_GROUPED_DEV, 16, true, true, 0, 0, "b200dpf_gen"},
    {MODE_FUSED_ET, MODE_EXPAND_ET, MODE_GROUPED_ET, MODE_GROUPED_ET_DEV, 8, true, false, 0, 0, "b200dpf_gen_et"},
    {MODE_FUSED_XOR, MODE_EXPAND_XOR, MODE_GROUPED_XOR, MODE_GROUPED_XOR_DEV, 4, false, false, 2, 4, "b200dpf_gen_xor"},
};

/* Trimmed tables (DESIGN.md section 11).  Row r of an n-row table sits at leaf position r >> lane_bits of a tree
 * over N = trimmed_domain(n) rows (the next power of two, at least the kind's n_min), so the live rows are a
 * prefix of the leaf positions and the work items past it are never issued. */
bool trim_args_ok(int64_t n, int kind) { return kind >= 0 && kind < host::KIND_COUNT && n >= 1 && n <= ((int64_t)1 << 31); }

int64_t trimmed_domain_of(int64_t n, int kind)
{
    return std::max<int64_t>((int64_t)1 << ilog2(n), host::kKinds[kind].n_min);
}

int64_t trimmed_alpha_of(int64_t row, int64_t n, int kind)
{
    const int b = host::kKinds[kind].lane_bits;
    return (int64_t)trimmed_alpha((uint64_t)row, ilog2(trimmed_domain_of(n, kind)) - b, b);
}

/* The shape of a table of n rows (bin < 0) or of bin `bin` for keys of `kind` (valid), or EINVAL for an n out of
 * range: a power of two in [n_min, 2^31], or when trimmed any n in [1, 2^31].  The device table is padded with
 * zero rows to a multiple of 2^g rows (one granule).  Untrimmed, that is the whole table.  Trimmed, one granule is
 * N/128 rows on a large table (the padding is then below N/128 < n/64) and never less than one work item of the
 * smallest size the launch planner keeps for the kind: 64 leaves of standard and early-terminated keys, 1 leaf
 * pair of XOR-shared ones (whose leaves are 128 rows of work).  Every issued item lies inside the padded rows. */
int table_shape(int64_t n, int kind, bool trimmed, int bin, TableShape *t)
{
    const host::KindInfo &k = host::kKinds[kind];
    if (trimmed ? !trim_args_ok(n, kind) : (n < k.n_min || n > ((int64_t)1 << 31) || (n & (n - 1)) != 0)) {
        char where[32] = "table";
        if (bin >= 0) snprintf(where, sizeof where, "bin %d:", bin);
        if (trimmed) return fail(B200DPF_EINVAL, "%s size n=%lld out of range [1, 2^31]", where, (long long)n);
        return fail(B200DPF_EINVAL, "%s size n=%lld must be a power of two in [%lld, 2^31]", where, (long long)n,
                    (long long)k.n_min);
    }
    const int log_n = ilog2(trimmed ? trimmed_domain_of(n, kind) : n);
    const int item_leaves_log2 = kKindOps[kind].leaf_items ? 1 : 6;
    const int g = trimmed ? std::min(log_n, std::max(log_n - 7, k.lane_bits + item_leaves_log2)) : log_n;
    *t = TableShape{n, log_n - k.lane_bits, (n + ((int64_t)1 << g) - 1) >> g << g, g - k.lane_bits, 0};
    return B200DPF_OK;
}

/* Where the rows of shape t live on the device, for shard `rank` of 2^shard_bits */
RowPlacement place_of(const TableShape &t, int lane_bits, bool trimmed, int rank, int shard_bits)
{
    return RowPlacement{t.first, (uint32_t)t.n, lane_bits, trimmed ? (int)PLACE_IDENTITY : t.depth - shard_bits,
                        (1u << shard_bits) - 1u, bitrev((uint32_t)rank, shard_bits), shard_bits};
}

/* "a standard", "an early-terminated", "an XOR-shared": the article of a kind's name */
inline const char *article(int kind) { return kind == host::KIND_STANDARD ? "a" : "an"; }

/* The refusal of entry point `name` of a key that is not of `kind` */
int fail_not_kind(int kind, const char *name)
{
    if (kind == host::KIND_STANDARD) return fail(B200DPF_EINVAL, "%s: malformed key", name);
    return fail(B200DPF_EINVAL, "%s: not an %s key", name, host::kKinds[kind].name);
}

/* Key number `b` of a batch (null: none) must be a key of the context's kind for its table, or its bin `bin` (>= 0),
 * of shape t: for n = 2^(t.depth + lane_bits) rows, the table's rows or trimmed_domain(rows).  Only a refused key is
 * decoded twice. */
int check_key(const b200dpf_ctx *c, const TableShape &t, const int32_t *key, int64_t b, int bin)
{
    const int kind = c->kind;
    const int64_t n = (int64_t)1 << (t.depth + c->lane_bits());
    const int64_t kn = key ? host::key_n(key, kind) : -1;
    if (kn == n) return B200DPF_OK;
    const int other = key ? host::key_kind(key) : -1;
    const host::KindInfo &k = host::kKinds[kind];
    char where[32] = "table";
    if (bin >= 0) snprintf(where, sizeof where, "bin %d", bin);
    if (kind == host::KIND_STANDARD && other > 0)
        return fail(B200DPF_EINVAL, "key %lld was generated for n=%lld, %s has n=%lld (it is %s %s key; this context takes standard keys)",
                    (long long)b, (long long)kn, where, (long long)n, article(other), host::kKinds[other].name);
    if (kind == host::KIND_STANDARD)
        return fail(B200DPF_EINVAL, "key %lld was generated for n=%lld, %s has n=%lld", (long long)b, (long long)kn, where, (long long)n);
    if (other >= 0 && other != kind)
        return fail(B200DPF_EINVAL, "key %lld is %s %s key; this %s context takes keys of %s", (long long)b, article(other),
                    host::kKinds[other].name, k.name, kKindOps[kind].gen);
    return fail(B200DPF_EINVAL, "key %lld is not %s %s key for n=%lld (its n: %lld)", (long long)b, article(kind), k.name,
                (long long)n, (long long)kn);
}

void fill_phase(const SmemLayout &L, int s, PhaseParams *ph)
{
    std::memset(ph, 0, sizeof *ph);
    ph->s = s;
    ph->stack_split = std::min(L.cap_lo, std::max(s - 1, 0));
}

/* What one run of the launcher evaluates, and where; its EvalPlan says how. */
struct EvalJob {
    const void *keys;
    KeyLayout kl;
    int64_t nkeys;
    int prf, mode_main;       /* mode_main: MODE_FUSED (out = [nkeys][entry_size] int32) or MODE_EXPAND (out = [nkeys][n] shares) */
    void *out;
    cudaStream_t stream;
    bool clear_out;           /* false: accumulate into out (b200dpf_eval_device_acc) */
    bool leaf_cache;          /* plain contexts, wide entries: cache the leaves, MAC-only passes for the other columns */
    /* grouped contexts: the key groups' descriptors and work units; `timed`: ev_t0 / ev_t1 bracket the launches */
    const GroupDesc *groups; const WorkUnit *units; uint32_t nunits;
    bool timed;
    const uint32_t *counts;   /* modes whose counts are on the device: EvalParams::dev_counts */
};

/*
 * How one evaluation (or one leaf-cache chunk of it) runs.  plan_eval (plain contexts) and plan_group_eval
 * (grouped ones) decide all of it from the context's shape, its knobs and the kernels' shared-memory
 * layouts, before anything is allocated or enqueued; launch_plan carries it out:
 *   one launch : [clear result + tickets, build frontier | grid barrier | main]  (+ passes, MAC passes)
 *   otherwise  : memset tickets, memset result, frontier kernel, main kernel x passes (+ MAC passes)
 */
struct EvalPlan {
    int mode, nv, passes;     /* main-phase kernel (MODE_*, uint4 columns per pass) and its passes over the columns */
    int kpw_log2;             /* log2 keys per warp */
    int64_t key_groups;
    int s;                    /* log2 leaves per main-phase work item (grouped: the largest of any key group) */
    int s_group;              /* grouped: a key group's s is this, within [1, its bin's depth] (group_s) */
    int f_rel, s_top;         /* frontier depth below the shard root, log2 leaves per tree-top item (0 = no frontier) */
    bool one_launch;          /* cooperative launches that clear their own accumulators before a grid barrier */
    bool grouped;             /* key groups of GroupDesc; no tree-top phase */
    bool leaf_cache, timing;  /* timing: per-block phase time stamps */
    bool tma_rows;            /* MODE_FUSED_TMA: each warp stages its item's rows in a tile after the stack */
    size_t tile_bytes;        /* all warps' tiles, then their mbarriers at off_tile_bar */
    uint32_t off_tile, off_tile_bar;
    SmemLayout L, LF;         /* main phase; tree-top phase (the stand-alone frontier kernel's unless one_launch) */
    size_t smem, smem_top;    /* dynamic shared memory of the main launches and of the frontier kernel */
    size_t pass_counters, top_counters;        /* main-phase tickets per pass; tree-top tickets (0: none) */
    size_t frontier_bytes, leaf_cache_bytes;
    PhaseParams main, top;    /* without their counters and frontier */
    uint32_t nfront, top_block_quota;          /* nfront: frontier nodes per key (this shard) */
    /* MAC-only passes: the cp.async.bulk variant or the register-staged one, its grid, position ranges per key group */
    bool mac_tma; int mac_grid; uint32_t mac_ranges;
};

/* The plan of one evaluation on a grouped context and its launch lists, made on the host in pinned staging and
 * uploaded on the caller's stream.  The uploads may still be pending when the call returns; ev_staged follows
 * them, and plan() waits for it on the host before it rewrites or regrows the staging. */
struct GroupLaunch {
    EvalPlan P;
    int64_t nkeys = 0, nunits = 0;
    PinnedBuffer<GroupDesc> h_descs;   /* the key groups' descriptors; all four lists hold at least 1,024 */
    DeviceBuffer<GroupDesc> d_descs;
    PinnedBuffer<WorkUnit> h_units;    /* modes that draw work units: the list */
    DeviceBuffer<WorkUnit> d_units;
    PinnedBuffer<uint2> h_order;       /* [nkeys] (caller's index, bin depth) by sorted position */
    DeviceBuffer<uint2> d_order;
    cudaEvent_t ev_staged = nullptr;
    bool staged_pending = false;
    ~GroupLaunch() { if (ev_staged) cudaEventDestroy(ev_staged); }
    int plan(b200dpf_ctx *c, int prf, const std::vector<int64_t> &count, const int32_t *bins);
    int upload(cudaStream_t stream, bool order);
};

/* The lists of b200dpf_group_eval_device_bins, planned on the device (dpf_group_plan.cu) into buffers of their own,
 * and the host half of their plan, which needs no key counts.  The host half is kept while nkeys, the prf and the
 * options stay those of the call that made it (b200dpf_ctx_set_option and _set_subtree_log2 clear `valid`). */
struct DevicePlanned {
    EvalPlan P;               /* key_groups: a bound of the key groups; s: the largest s a group can be given */
    int64_t nkeys = 0;
    int64_t units_bound = 0;
    int prf = -1;
    bool valid = false;
    GroupPlanParams gp{};     /* without the caller's bins and bad-key word */
    DeviceBuffer<uint32_t> d_hist, d_sort, d_counts;   /* d_sort: keys in, keys out, values in, values out */
    DeviceBuffer<void> d_temp;
    DeviceBuffer<uint4> d_bin_first;
    DeviceBuffer<uint2> d_order;
    DeviceBuffer<GroupDesc> d_descs;
    DeviceBuffer<WorkUnit> d_units;
};

}  // namespace

struct GroupBins {
    std::vector<TableShape> shape;     /* [nbins] */
    /* made at create, never rewritten: [nbins] the bins' placements, for row updates and the key generator; [nbins]
     * (uint4 offset of bin g's key in a compact query, depth of g), with query_v uint4 per query; the key generator's
     * AES table */
    DeviceBuffer<RowPlacement> d_place;
    DeviceBuffer<uint2> d_bins;
    uint64_t query_v = 0;
    DeviceBuffer<uint32_t> d_te0;
    DeviceBuffer<GroupBinInfo> d_bin_info;   /* made at create, never rewritten: [nbins] what the device planner reads */
    GroupLaunch once;                  /* b200dpf_group_eval and _eval_device: planned by every call */
    /* b200dpf_group_eval_queries_device: kept while nq, the prf and the options stay those of the call that made
     * it (b200dpf_ctx_set_option and _set_subtree_log2 clear cached_valid) */
    GroupLaunch cached;
    int64_t cached_nq = 0;
    int cached_prf = -1;
    bool cached_valid = false;
    DevicePlanned device_planned;      /* b200dpf_group_eval_device_bins */
    /* a batch-code context (b200dpf_batchcode_create): the layout its bins follow.  Its rows change only three
     * copies at a time (b200dpf_batchcode_update_rows), so b200dpf_group_update_rows refuses it. */
    std::optional<BatchCodeLayout> batch;
    /* a keyword-PIR context (b200dpf_kwpir_create): the layout its three bins follow, and the rounds its placement
     * took and their device time.  A row update could overwrite a tag, so b200dpf_group_update_rows refuses it. */
    struct Keyword {
        KeywordLayout layout;
        int rounds;
        float place_ms;
    };
    std::optional<Keyword> keyword;
};

namespace {

/* Work-item size: from s down to s_floor, the first s at which the launch has at least `wanted` items */
template <class Items> int shrink_s(int s, int s_floor, int64_t wanted, Items items)
{
    while (s > s_floor && items(s) < wanted) s--;
    return s;
}

/* The work-item size of a key group of bin g on a grouped context */
int group_s(const EvalPlan &P, const GroupBins &B, int g) { return std::max(1, std::min(B.shape[(size_t)g].room, P.s_group)); }

/* The fields of EvalParams that every launch of job J on layout L shares; the others are zero. */
void fill_common(const b200dpf_ctx *c, const SmemLayout &L, const EvalJob &J, const EvalPlan &P, EvalParams *p)
{
    std::memset(p, 0, sizeof *p);
    p->keys = reinterpret_cast<const uint4 *>(J.keys);
    p->key_stride_v = J.kl.stride_v; p->key_root_v = J.kl.root_v; p->key_compact = J.kl.compact;
    p->depth = c->shape.depth;
    p->nkeys = (int)J.nkeys; p->kpw_log2 = P.kpw_log2; p->key_groups = (int)P.key_groups;
    p->groups = J.groups; p->units = J.units; p->nunits = J.nunits; p->dev_counts = J.counts;
    p->table = reinterpret_cast<const uint4 *>(c->d_table.ptr);
    p->row_stride_v = (uint32_t)c->entry_pad / 4u;
    p->out_stride = (uint32_t)c->entry_size;
    p->n = (uint64_t)c->shape.n;
    p->off_cw = L.off_meta;
    p->off_cwlo = L.off_small;
    p->off_root = p->off_cwlo + 512u;
    p->off_flag = p->off_root + 512u;
    p->off_stack_lo = L.off_lo;
    p->off_stack_hi = L.off_hi;
    p->off_tab = L.off_tab;
}

/* The plan of job J on a plain context. */
int plan_eval(b200dpf_ctx *c, const EvalJob &J, EvalPlan *out)
{
    const b200dpf_ctx::Knobs &K = c->knobs;
    const KindOps &ops = kKindOps[c->kind];
    const int prf = J.prf;
    const int64_t nkeys = J.nkeys;
    const bool fused = J.mode_main == MODE_FUSED;
    EvalPlan &P = *out = EvalPlan{};
    int &kpw_log2 = P.kpw_log2, &s = P.s, &f_rel = P.f_rel, &s_top = P.s_top;   /* the names the arithmetic below uses */
    int64_t &key_groups = P.key_groups;
    SmemLayout &L = P.L;
    P.leaf_cache = J.leaf_cache;
    /* Entries wider than 32 columns: the tree is expanded ONCE by the best-shaped kernel (16
     * columns, NV = 4), which also caches each leaf's low word; every other column is produced by
     * MAC-only passes over that cache.  Without the cache (disabled or lane-split batches) wide
     * entries use one tree expansion per 64 columns. */
    P.nv = (!fused || c->entry_pad <= 16 || P.leaf_cache) ? 4 : std::min(ops.max_nv, c->entry_pad <= 32 ? 8 : 16);
    P.passes = fused ? (P.leaf_cache ? 1 : c->entry_pad / (4 * P.nv)) : 1;
    /* optional variant: the rows of each work item staged into shared memory by cp.async.bulk */
    P.tma_rows = K.tma_rows != 0 && K.one_launch != 0 && c->coop_ok != 0 && fused && c->entry_pad == 16 &&
                 prf != B200DPF_PRF_AES128 && nkeys >= 17 && ops.tma_rows;
    const int mode_plain = fused ? ops.mode_fused : ops.mode_expand;
    P.mode = P.tma_rows ? MODE_FUSED_TMA : mode_plain;
    /* keys per warp: a full warp of keys when the batch allows; for small batches the
     * spare lanes take adjacent subtrees of the same keys (single-query latency mode) */
    kpw_log2 = 5;
    if (K.lane_split != 0)
        while (kpw_log2 > 0 && ((int64_t)1 << (kpw_log2 - 1)) >= nkeys) kpw_log2--;
    if (fused) kpw_log2 = std::max(kpw_log2, ops.min_kpw_log2);
    key_groups = (nkeys + ((int64_t)1 << kpw_log2) - 1) >> kpw_log2;
    /* AES binds the shared-memory data pipe, and a broadcast row load is charged for every lane's copy
     * of the row: with at least 4 keys per warp, each lane of a key quad loads a quarter of the row and
     * the quad trades leaf values by SHFL instead (DESIGN.md section 3).  Decided before the layout: the
     * kernel runs more threads, so its stack holds fewer levels (s_max).  kpw_log2 only grows below. */
    if (P.mode == MODE_FUSED && prf == B200DPF_PRF_AES128 && P.nv == 4 && kpw_log2 >= 2)
        P.mode = MODE_FUSED_COLSPLIT;
    int rc = smem_layout(c, prf, P.nv, P.mode, &L);
    if (rc) return rc;
    const int64_t warps = (int64_t)L.grid * (L.threads / 32);

    /* ---- work-item size s and the frontier depth --------------------------------
     * Without a frontier every item re-walks depth-s levels from the root, so items
     * must be big; with one the walk is (almost) free and small items balance the
     * tail. */
    const bool want_frontier = K.frontier != 0;
    if (K.subtree_log2 > 0) {
        s = std::min(K.subtree_log2, std::min(c->depth_local(), L.s_max));
    } else {
        /* B=512 E=16, frontier on, 1x H100 SXM 80 GB at a 400 W power limit, DPFs/s (run-to-run
         * spread about 3 %); the automatic choice is within the spread of the best fixed s:
         *   AES n=2^20: auto 19.47k; s=4 19.39k, 5 19.77k, 6 19.56k, 7 20.01k, 8 19.56k
         *   AES n=2^16: auto 319.3k; s=4 317.5k, 5 318.1k, 6 318.1k, 7 300.5k
         *   ChaCha n=2^20: auto 19.18k; s=5 18.94k, 6 19.13k, 7 19.19k */
        const int s_cap = want_frontier ? 7 : ((prf == B200DPF_PRF_AES128) ? 8 : 10);
        /* XOR-shared keys: a leaf is 128 rows of work, so a few items per warp balance the tail and the
         * smallest items keep every warp busy at small n.  AES, E=16, B=512, H100 80GB HBM3 at a 700 W
         * power limit, SM clock 1980 MHz, ms per batch (DESIGN.md section 10):
         *   n=2^16: auto 0.107; s=1 0.103, 2 0.148, 3 0.196, 4 0.262, 5 0.490
         *   n=2^20: auto 0.971; s=1 0.989, 2 0.980, 3 0.971, 4 0.975, 5 0.975, 6 0.973 */
        const int s_floor = ops.leaf_items ? 1 : want_frontier ? 3 : 5;
        const int64_t items_per_warp = ops.leaf_items ? ops.leaf_items : want_frontier ? 24 : 6;
        s = shrink_s(std::min(c->depth_local(), std::min(L.s_max, s_cap)), s_floor, items_per_warp * warps, [&](int t) {
            return ((c->rows_local() >> (t + c->lane_bits())) * key_groups) >> (5 - kpw_log2);
        });
    }
    if (s < 1) s = 1;
    if (P.tma_rows) {
        /* one tile of 2^s 64-byte rows per warp, after the sibling stack */
        const int warps_blk = L.threads / 32;
        if (K.subtree_log2 <= 0) s = std::min(s, 6);
        P.tile_bytes = (size_t)warps_blk * ((size_t)64 << s) + 8u * (size_t)warps_blk + 16u;
        if ((size_t)L.off_lo + (size_t)(std::max(s, 7) - 1) * L.level_bytes + P.tile_bytes > (size_t)L.budget) {
            P.tma_rows = false;             /* does not fit beside correction words and stack: broadcast loads */
            P.mode = mode_plain;
            P.tile_bytes = 0;
            rc = smem_layout(c, prf, P.nv, P.mode, &L);
            if (rc) return rc;
        }
    }
    if (c->trimmed) {
        /* a ticket (2^(s + spw_log2) leaves) must not reach past the padded rows: smaller items first (down to
         * one leaf pair), then fewer subtrees per warp.  Lanes of a key quad trade leaf values by SHFL, so every
         * lane of an issued ticket runs; the padding is what keeps its rows inside the table. */
        const int room = c->shape.room;
        s = std::max(1, std::min(s, room - (5 - kpw_log2)));
        if (5 - kpw_log2 > room - s) {
            kpw_log2 = 5 - (room - s);
            key_groups = (nkeys + ((int64_t)1 << kpw_log2) - 1) >> kpw_log2;
        }
    }
    const int rel = c->depth_local() - s;           /* tree levels between the shard root and the items */
    if (5 - kpw_log2 > rel) {                     /* not enough subtrees to split a warp that far */
        kpw_log2 = 5 - rel;
        key_groups = (nkeys + ((int64_t)1 << kpw_log2) - 1) >> kpw_log2;
    }
    const int spw_log2 = 5 - kpw_log2;
    if (P.leaf_cache && kpw_log2 != 5) return fail(B200DPF_ESTATE, "internal: leaf cache planned for a lane-split batch");

    if (want_frontier && rel >= 2) {
        const int64_t cap_bytes = (int64_t)K.frontier_mb << 20;
        f_rel = rel;
        while (f_rel > 0 && ((key_groups * (16 << kpw_log2)) << f_rel) > cap_bytes) f_rel--;
        if (f_rel < 2 || f_rel < spw_log2 + 1) f_rel = 0;
    }

    P.one_launch = K.one_launch != 0 && c->coop_ok != 0;
    P.pass_counters = (size_t)key_groups;
    P.top_counters = std::max<size_t>((size_t)key_groups, 64);
    if (f_rel > 0) P.frontier_bytes = ((size_t)key_groups * (16 << kpw_log2)) << f_rel;

    /* ---- the tree-top phase (frontier build) ---- */
    P.LF = L;
    if (f_rel > 0) {
        if (!P.one_launch && (rc = smem_layout(c, prf, 4, MODE_FRONTIER, &P.LF))) return rc;
        const SmemLayout &LF = P.LF;
        s_top = std::max(1, std::min(f_rel - spw_log2, std::min(5, LF.s_max)));
        if (K.top_log2 > 0) {
            s_top = std::max(1, std::min(K.top_log2, std::min(f_rel - spw_log2, LF.s_max)));
        } else if (P.one_launch && K.balance_top) {
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
        fill_phase(LF, s_top, &P.top);
        P.top.nsub = (uint32_t)1 << (f_rel - s_top);
        P.top.sub_first = (uint32_t)c->shard_rank << (f_rel - s_top);
        P.top.walk_first_level = c->shape.depth - 1;
        P.top.walk_steps = c->shard_bits + f_rel - s_top;
        P.top.level_base = c->depth_local() - f_rel;
        P.smem_top = smem_bytes(LF, s_top);
        P.nfront = (uint32_t)1 << f_rel;
    }

    /* ---- the main phase ---- */
    P.smem = smem_bytes(L, std::max(s, s_top));
    if (P.tma_rows) {
        P.off_tile = (uint32_t)((P.smem + 15) & ~(size_t)15);
        P.off_tile_bar = P.off_tile + (uint32_t)((size_t)(L.threads / 32) * ((size_t)64 << s));
        P.smem = (size_t)P.off_tile + P.tile_bytes;
    }
    fill_phase(L, s, &P.main);
    P.main.nsub = (uint32_t)(c->rows_local() >> (s + c->lane_bits()));   /* 2^rel, or the items over a trimmed table's rows */
    P.main.sub_first = (uint32_t)c->shard_rank << rel;
    if (f_rel > 0) {
        P.main.front_shift = rel - f_rel;
        P.main.walk_first_level = c->depth_local() - f_rel - 1;
        P.main.walk_steps = rel - f_rel;
    } else {
        P.main.walk_first_level = c->shape.depth - 1;
        P.main.walk_steps = c->shape.depth - s;
    }
    if (P.one_launch) {
        const uint64_t items = (uint64_t)key_groups * (uint64_t)(P.top.nsub >> spw_log2);
        P.top_block_quota = K.balance_top ? (uint32_t)std::max<uint64_t>(1, (items + (uint64_t)L.grid - 1) / (uint64_t)L.grid)
                                          : 0x7fffffffu;
        P.timing = K.timing != 0;
    }

    /* ---- wide entries: the leaf-caching pass, then the MAC-only passes ---- */
    if (P.leaf_cache) {
        P.mode = ops.mode_fused;                   /* the kind's fused kernel, on the layout planned above */
        P.leaf_cache_bytes = (size_t)key_groups * 32u * (size_t)c->rows_local() * sizeof(uint32_t);
        P.mac_tma = K.mac_tma != 0;
        /* register-staged variant: 8 warps per block */
        const int64_t mac_warps = (int64_t)c->sm_count * 2 * 8;
        const int64_t ranges = std::max<int64_t>(1, (2 * mac_warps + key_groups - 1) / key_groups);
        /* TMA variant: one block per SM; a block takes 8 key groups x one position range */
        const int64_t kg_blocks = (key_groups + 7) / 8;
        const int64_t tr = std::max<int64_t>(1, (2 * (int64_t)c->sm_count + kg_blocks - 1) / kg_blocks);
        P.mac_grid = P.mac_tma ? c->sm_count : c->sm_count * 2;
        P.mac_ranges = (uint32_t)(P.mac_tma ? std::min<int64_t>(tr, std::max<int64_t>(1, c->rows_local() / 256))
                                            : std::min<int64_t>(ranges, std::max<int64_t>(1, c->rows_local() / 64)));
    }
    return B200DPF_OK;
}

/* The part of a grouped plan that needs no key counts: the mode, the passes, the shared-memory layout and the grid
 * (which depend on the kernel alone, not on s), and s_group before shrink_s.  Automatic s (`shrink`) shrinks it from
 * there down to *s_floor while the launch has fewer than *items_wanted work items. */
int plan_group_base(b200dpf_ctx *c, int prf, int mode, EvalPlan *out, bool *shrink, int *s_floor, int64_t *items_wanted)
{
    const KindOps &ops = kKindOps[c->kind];
    EvalPlan &P = *out = EvalPlan{};
    const SmemLayout &L = P.L;
    P.grouped = P.one_launch = true;
    P.mode = mode;
    P.nv = 4; P.passes = c->entry_pad / 16;     /* 16 columns per pass */
    P.kpw_log2 = 5;
    int rc = smem_layout(c, prf, P.nv, P.mode, &P.L);
    if (rc) return rc;
    const int64_t warps = (int64_t)L.grid * (L.threads / 32);
    P.s_group = std::min(c->knobs.subtree_log2 > 0 ? c->knobs.subtree_log2 : 6, L.s_max);
    *shrink = c->knobs.subtree_log2 <= 0;
    *s_floor = ops.leaf_items ? 1 : 3;
    *items_wanted = (ops.leaf_items ? ops.leaf_items : 2) * warps;
    return B200DPF_OK;
}

/* The plan of one evaluation on a grouped context, whose bin-sorted keys of bin g are at positions
 * count[g] .. count[g + 1].  Key groups and their work-item size: big items amortise the root-to-subtree
 * walk every item pays (there is no frontier: bins are small), small items keep every warp busy.  Leaves
 * of many rows (KindOps::leaf_items) take items down to s = 1, as on a plain context.  One cooperative
 * launch per 16 columns; the first one clears the result and every pass's tickets. */
int plan_group_eval(b200dpf_ctx *c, int prf, const std::vector<int64_t> &count, EvalPlan *out)
{
    const GroupBins *B = c->bins.get();
    const int nbins = (int)B->shape.size();
    EvalPlan &P = *out;
    const SmemLayout &L = P.L;
    bool shrink = false;
    int s_floor = 0;
    int64_t items_wanted = 0;
    int rc = plan_group_base(c, prf, kKindOps[c->kind].mode_grouped, out, &shrink, &s_floor, &items_wanted);
    if (rc) return rc;
    auto groups_of = [&](int g) { return (count[(size_t)g + 1] - count[(size_t)g] + 31) / 32; };
    for (int g = 0; g < nbins; g++) P.key_groups += groups_of(g);
    if (shrink) {
        P.s_group = shrink_s(P.s_group, s_floor, items_wanted, [&](int t) {
            int64_t items = 0;
            for (int g = 0; g < nbins; g++)
                items += groups_of(g) * (B->shape[(size_t)g].rows >> (std::min(B->shape[(size_t)g].room, t) + c->lane_bits()));
            return items;
        });
    }
    P.s = 1;
    for (int g = 0; g < nbins; g++)
        if (count[(size_t)g + 1] > count[(size_t)g]) P.s = std::max(P.s, group_s(P, *B, g));
    /* per pass: one ticket counter per key group, or the one unit counter */
    P.pass_counters = mode_traits(P.mode).units ? 1u : (size_t)P.key_groups;
    P.smem = smem_bytes(L, P.s);
    fill_phase(L, P.s, &P.main);
    return B200DPF_OK;
}

/* The host half of the plan of b200dpf_group_eval_device_bins for nkeys keys: plan_group_base, bounds of the lists
 * the device half writes, and their buffers.  The rest (the counts, s_group, every group's s, the lists) is
 * computed on the device from the bins by launch_group_plan. */
int plan_group_device(b200dpf_ctx *c, int prf, int64_t nkeys, DevicePlanned *D)
{
    GroupBins *B = c->bins.get();
    const int nbins = (int)B->shape.size();
    EvalPlan &P = D->P;
    const SmemLayout &L = P.L;
    D->valid = false;
    bool shrink = false;
    int s_floor = 0;
    int64_t items_wanted = 0;
    int rc = plan_group_base(c, prf, kKindOps[c->kind].mode_grouped_dev, &P, &shrink, &s_floor, &items_wanted);
    if (rc) return rc;
    /* every key group but the last of its bin holds 32 keys: at most nkeys / 32 full groups, and one partial group
     * per bin that has keys */
    P.key_groups = nkeys / 32 + std::min<int64_t>(nbins, nkeys);
    /* shared memory for the largest s a group can be given (group_s <= max(1, s_group)); a group's own s only picks
     * its items.  L.grid and the block shape come from the kernel alone, so they do not depend on s. */
    P.s = std::max(1, P.s_group);
    P.pass_counters = mode_traits(P.mode).units ? 1u : (size_t)P.key_groups;
    P.smem = smem_bytes(L, P.s);
    fill_phase(L, P.s, &P.main);
    /* Work units (GroupLaunch::plan): a key group of nsub items is cut into ceil(nsub / per_unit) units, per_unit =
     * clamp(ceil(items / grid), 1, W) with W warps per block and `items` the sum of every group's nsub.  So units
     * <= key groups + items / per_unit.  While per_unit < W, per_unit >= items / grid and items / per_unit <= grid;
     * at per_unit = W, items / W <= key groups * nsub_max / W, nsub_max being the most items a bin's group can
     * have (at s = 1). */
    const bool units = mode_traits(P.mode).units;
    const int unit_cap = L.threads / 32;
    D->units_bound = 0;
    if (units) {
        int64_t nsub_max = 1;
        for (const TableShape &t : B->shape) nsub_max = std::max<int64_t>(nsub_max, t.rows >> (1 + c->lane_bits()));
        D->units_bound = P.key_groups + std::max<int64_t>(L.grid, (P.key_groups * nsub_max + unit_cap - 1) / unit_cap);
    }
    GroupPlanParams &g = D->gp;
    g = GroupPlanParams{};
    g.nkeys = nkeys;
    g.nbins = nbins;
    g.bin_info = B->d_bin_info.ptr;
    g.lane_bits = c->lane_bits();
    g.s_start = P.s_group;
    g.shrink = shrink ? 1 : 0;
    g.s_floor = s_floor;
    g.items_wanted = items_wanted;
    g.units = units ? 1 : 0;
    g.grid = L.grid;
    g.unit_cap = unit_cap;
    g.end_bit = ilog2((int64_t)nbins + 1);     /* sort keys 0 .. nbins, nbins for a key outside every bin */
    CUDA_TRY(group_plan_temp_bytes(nkeys, g.end_bit, &g.temp_bytes));
    g.descs_cap = P.key_groups;
    g.units_cap = D->units_bound;
    rc = D->d_hist.reserve(((size_t)nbins + 1) * sizeof(uint32_t));
    if (!rc) rc = D->d_counts.reserve(4 * sizeof(uint32_t));
    if (!rc) rc = D->d_bin_first.reserve((size_t)nbins * sizeof(uint4));
    if (!rc) rc = D->d_sort.reserve(4 * (size_t)nkeys * sizeof(uint32_t));
    if (!rc) rc = D->d_temp.reserve(std::max<size_t>(g.temp_bytes, 1));
    if (!rc) rc = D->d_order.reserve((size_t)nkeys * sizeof(uint2));
    if (!rc) rc = D->d_descs.reserve((size_t)P.key_groups * sizeof(GroupDesc));
    if (!rc && units) rc = D->d_units.reserve((size_t)D->units_bound * sizeof(WorkUnit));
    if (rc) return rc;
    g.hist = D->d_hist.ptr;
    g.keys_in = D->d_sort.ptr;
    g.keys_out = g.keys_in + nkeys;
    g.vals_in = g.keys_out + nkeys;
    g.vals_out = g.vals_in + nkeys;
    g.temp = D->d_temp.ptr;
    g.bin_first = D->d_bin_first.ptr;
    g.order = D->d_order.ptr;
    g.descs = D->d_descs.ptr;
    g.units_out = D->d_units.ptr;
    g.counts = D->d_counts.ptr;
    D->nkeys = nkeys;
    D->prf = prf;
    D->valid = true;
    return B200DPF_OK;
}

/* Carry out plan P of job J: reserve what it asks for, order it after the context's last operation, clear,
 * launch and make that the context's last operation.  A device that cannot keep the whole persistent grid
 * resident (a partitioned GPU, say) refuses the first cooperative launch before anything of the evaluation
 * ran: a plain context then falls back, for its life, to separate launches, planned again. */
int launch_plan(b200dpf_ctx *c, const EvalJob &J, const EvalPlan &P)
{
    const bool fused = J.mode_main == MODE_FUSED;
    const size_t n_counters = (size_t)P.passes * P.pass_counters;
    bool grown = false;
    int rc = c->d_counters.reserve(n_counters * sizeof(uint32_t));
    if (!rc && P.top_counters) rc = c->d_top_counters.reserve(P.top_counters * sizeof(uint32_t), &grown);
    if (grown) c->coop_state_dirty = true;
    if (!rc && P.frontier_bytes) rc = c->d_frontier.reserve(P.frontier_bytes);
    if (!rc) rc = wait_last(c, J.stream);
    if (rc) return rc;

    if (!P.one_launch || c->coop_state_dirty) {
        if (P.top_counters) CUDA_TRY(cudaMemsetAsync(c->d_top_counters.ptr, 0, c->d_top_counters.cap, J.stream));
        CUDA_TRY(cudaMemsetAsync(c->d_gridbar.ptr, 0, sizeof(uint32_t), J.stream));
        c->bar_epoch = 0;
        c->coop_state_dirty = false;
    }
    if (!P.one_launch) {
        CUDA_TRY(cudaMemsetAsync(c->d_counters.ptr, 0, n_counters * sizeof(uint32_t), J.stream));
        if (fused && J.clear_out)
            CUDA_TRY(cudaMemsetAsync(J.out, 0, (size_t)J.nkeys * c->entry_size * sizeof(int32_t), J.stream));
        c->coop_state_dirty = true;     /* the stand-alone frontier kernel leaves its tickets used */
    }
    if (P.timing) rc = c->d_timing.reserve((size_t)P.L.grid * 8 * sizeof(unsigned long long));
    if (!rc && P.leaf_cache_bytes) rc = c->d_leaf_cache.reserve(P.leaf_cache_bytes);
    if (rc) return rc;
    if (P.timing) CUDA_TRY(cudaMemsetAsync(c->d_timing.ptr, 0, c->d_timing.cap, J.stream));
    c->last_launches = 0;
    if (J.timed) CUDA_TRY(cudaEventRecord(c->ev_t0, J.stream));

    EvalParams p;
    PhaseParams top = P.top;
    if (P.f_rel > 0) top.counters = c->d_top_counters.ptr;
    uint4 *const frontier = reinterpret_cast<uint4 *>(c->d_frontier.ptr);
    if (P.f_rel > 0 && !P.one_launch) {           /* the stand-alone frontier kernel */
        fill_common(c, P.LF, J, P, &p);
        p.main = top; p.nfront = P.nfront; p.frontier_out = frontier;
        CUDA_TRY(launch_eval(J.prf, 4, MODE_FRONTIER, p, P.LF.grid, P.smem_top, J.stream));
        c->last_launches++;
    }

    fill_common(c, P.L, J, P, &p);
    p.main = P.main;
    p.main.counters = c->d_counters.ptr;
    if (P.f_rel > 0) p.main.frontier_in = frontier;
    p.nfront = P.nfront;
    p.off_tile = P.off_tile; p.off_tile_bar = P.off_tile_bar;
    if (P.one_launch) {
        p.fuse_top = 1;
        if (fused && J.clear_out) { p.zero_a = reinterpret_cast<uint32_t *>(J.out); p.zero_a_words = (uint64_t)J.nkeys * c->entry_size; }
        p.zero_b = c->d_counters.ptr; p.zero_b_words = n_counters;
        if (!P.grouped) {
            p.top = top;                  /* nsub == 0: no frontier, the top phase only clears */
            p.frontier_out = frontier;
            p.rearm = c->d_top_counters.ptr; p.rearm_words = (uint32_t)P.key_groups;
            p.top_block_quota = P.top_block_quota;
        }
        if (P.timing) p.timing = c->d_timing.ptr;
        p.grid_bar = c->d_gridbar.ptr;
        c->bar_epoch += (uint32_t)P.L.grid;
        p.grid_bar_target = c->bar_epoch;
    }

    bool coop_refused = false;
    auto launch_main = [&]() -> int {
        const cudaError_t e = launch_eval(J.prf, P.nv, P.mode, p, P.L.grid, P.smem, J.stream);
        if (e != cudaSuccess) {
            c->coop_state_dirty = true;
            coop_refused = e == cudaErrorCooperativeLaunchTooLarge && p.fuse_top && !P.grouped;
            return fail(B200DPF_ECUDA, "%s: %s", P.grouped ? "grouped evaluation launch" : "evaluation kernel launch",
                        cudaGetErrorString(e));
        }
        c->last_launches++;
        p.fuse_top = 0;                   /* later passes of this evaluation reuse the frontier */
        return B200DPF_OK;
    };
    if (J.mode_main == MODE_EXPAND) {
        p.shares = reinterpret_cast<uint32_t *>(J.out);
        rc = launch_main();
    } else {
        p.out = reinterpret_cast<uint32_t *>(J.out);
        if (P.leaf_cache) { p.leaf_cache = c->d_leaf_cache.ptr; p.n_local = (uint64_t)c->rows_local(); }
        for (int pass = 0; pass < P.passes && rc == B200DPF_OK; pass++) {
            p.col_off_v = (uint32_t)(pass * P.nv);
            p.col_off = (uint32_t)(pass * 4 * P.nv);
            p.ncols = (uint32_t)std::max(0, std::min(4 * P.nv, c->entry_size - pass * 4 * P.nv));
            if (p.ncols == 0) break;
            p.main.counters = c->d_counters.ptr + (size_t)pass * P.pass_counters;
            rc = launch_main();
        }
    }
    if (coop_refused) {
        cudaGetLastError();
        c->coop_ok = 0;
        EvalPlan Q;
        return (rc = plan_eval(c, J, &Q)) ? rc : launch_plan(c, J, Q);
    }
    if (rc) return rc;

    if (P.leaf_cache) {
        MacParams m;
        std::memset(&m, 0, sizeof m);
        m.leaf_cache = p.leaf_cache; m.table = p.table; m.row_stride_v = p.row_stride_v;
        m.out = p.out; m.out_stride = p.out_stride;
        m.nkeys = (int)J.nkeys; m.key_groups = (int)P.key_groups; m.n_local = (uint64_t)c->rows_local();
        m.ranges_per_group = P.mac_ranges;
        for (int blk = 0; blk * 64 < c->entry_size; blk++) {       /* 64-column slices of the rows */
            m.col_off_v = (uint32_t)(blk * 16); m.col_off = (uint32_t)(blk * 64);
            m.ncols = (uint32_t)std::min(64, c->entry_size - blk * 64);
            m.col_skip = blk == 0 ? 16u : 0u;                      /* columns 0..15 came from the fused pass */
            if (m.ncols <= m.col_skip) continue;
            if (P.mac_tma) CUDA_TRY(launch_mac_tma(m, P.mac_grid, J.stream));
            else CUDA_TRY(launch_mac(16, m, P.mac_grid, J.stream));
            c->last_launches++;
        }
    }
    if (J.timed) { CUDA_TRY(cudaEventRecord(c->ev_t1, J.stream)); c->timed = true; }
    return mark_last(c, J.stream);
}

/*
 * One evaluation on a plain context.  Wide entries whose leaf cache (nkeys x rows_local x 4 bytes) would
 * exceed the cap are evaluated in batch chunks that fit -- the cache is what makes columns beyond the
 * first 16 cost a MAC pass instead of a tree expansion, so shrinking the chunk beats dropping the cache.
 */
int run_pipeline(b200dpf_ctx *c, const void *keys_dev, const KeyLayout &kl, int64_t nkeys, int prf, int mode_main,
                 void *out_dev, cudaStream_t stream, bool clear_out = true)
{
    const b200dpf_ctx::Knobs &K = c->knobs;
    const bool wide = mode_main == MODE_FUSED && c->entry_pad > 32 && nkeys >= 17 && K.leaf_cache != 0 && kKindOps[c->kind].leaf_cache;
    const size_t per_group = 32u * (size_t)c->rows_local() * sizeof(uint32_t);
    const size_t cap = (size_t)std::max(K.leaf_cache_mb, 1) << 20;
    /* not a cached evaluation, or one key group alone overflows the cap (re-expand per 64 columns): one chunk */
    const bool cached = wide && per_group <= cap;
    const int64_t chunk = cached ? (int64_t)std::max<size_t>(1, cap / per_group) * 32 : nkeys;
    EvalJob J{keys_dev, kl, nkeys, prf, mode_main, out_dev, stream, clear_out};
    int rc = B200DPF_OK, launches = 0;
    for (int64_t k0 = 0; k0 < nkeys && rc == B200DPF_OK; k0 += chunk) {
        J.nkeys = std::min(chunk, nkeys - k0);
        J.keys = reinterpret_cast<const char *>(keys_dev) + (size_t)k0 * kl.stride_v * 16u;
        J.out = reinterpret_cast<char *>(out_dev) + (size_t)k0 * c->entry_size * sizeof(int32_t);
        /* a ragged tail below 17 keys would be lane-split, which the cache layout excludes */
        J.leaf_cache = cached && J.nkeys >= 17;
        EvalPlan P;
        rc = plan_eval(c, J, &P);
        if (!rc) rc = launch_plan(c, J, P);
        launches += c->last_launches;
    }
    c->last_launches = launches;
    return rc;
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
    /* the environment is consulted here and nowhere else (b200dpf_ctx_set_option changes a live context) */
    if (read_env)
        for (const KnobInfo &k : kKnobs) c->knobs.*k.field = env_int(k.env, k.dflt);
    CUDA_TRY(probe_dynamic_smem_base(&c->smem_base, c->stream));
    CUDA_TRY(upload_aes_table(host::aes_te0()));
    *out = std::move(c);
    return B200DPF_OK;
}

/* Whether `src` is device memory (then *src_device is its device), after waiting for that device: the caller's table
 * may still be being written there. */
int wait_source(const b200dpf_ctx *c, const void *src, bool *on_device, int *src_device)
{
    cudaPointerAttributes attr;
    *on_device = cudaPointerGetAttributes(&attr, src) == cudaSuccess &&
                 (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
    cudaGetLastError();
    *src_device = *on_device ? attr.device : -1;
    if (*on_device) {  /* it may still be being written on the caller's stream (e.g. a dtype cast enqueued just before
                        * this call): our copy runs on a private non-blocking stream, so wait for its device first */
        if (attr.device != c->device) cudaSetDevice(attr.device);
        const cudaError_t es = cudaDeviceSynchronize();
        if (attr.device != c->device) cudaSetDevice(c->device);
        CUDA_TRY(es);
    }
    return B200DPF_OK;
}

/* Bytes of the device stage that carries a caller's rows to their context when they cannot be read in place */
constexpr size_t kStageBytes = (size_t)64 << 20;

/* Write the caller's rows into c's device table and wait; any stream may read the table on return.  `src` holds `rows`
 * rows of `cols` int32 in host or device memory, of which c owns all, or with own.shift > 0 those of one shard: the leaves
 * own.own_val + k * 2^own.shift, 2^own.lane_bits rows each.  scatter(chunk, first, count) enqueues on c->stream the
 * kernel that places own rows [first, first + count), which chunk holds as [count][cols].  A contiguous source on c's
 * device is read in place; any other goes through one device stage of at most kStageBytes, a whole number of leaves at
 * a time.  A caller that writes several tables passes `keep`, the stage they share, so that it is allocated once. */
template <class Scatter>
int write_rows(b200dpf_ctx *c, const int32_t *src, uint64_t rows, int cols, const RowPlacement &own, Scatter scatter,
               DeviceBuffer<int32_t> *keep = nullptr)
{
    bool on_device;
    int src_device;
    int rc = wait_source(c, src, &on_device, &src_device);
    if (rc) return rc;
    const uint64_t own_rows = rows >> own.shift;
    DeviceBuffer<int32_t> local;
    DeviceBuffer<int32_t> &stage = keep ? *keep : local;
    if (own.shift == 0 && on_device && src_device == c->device) {
        CUDA_TRY(scatter(src, 0, own_rows));
    } else {
        const size_t row_bytes = (size_t)cols * sizeof(int32_t), leaf_bytes = row_bytes << own.lane_bits;
        const uint64_t chunk = std::min<uint64_t>(own_rows, std::max<size_t>(1, kStageBytes / leaf_bytes) << own.lane_bits);
        rc = stage.reserve((size_t)chunk * row_bytes);
        if (rc) return rc;
        for (uint64_t r0 = 0; r0 < own_rows; r0 += chunk) {     /* one stream: a chunk's copy waits for the previous scatter */
            const uint64_t count = std::min<uint64_t>(chunk, own_rows - r0);
            if (own.shift == 0) {
                CUDA_TRY(cudaMemcpyAsync(stage.ptr, src + r0 * (uint64_t)cols, (size_t)count * row_bytes, cudaMemcpyDefault, c->stream));
            } else {   /* own row r0 starts natural row (r0 << shift) + (own_val << lane_bits) */
                const int32_t *from = src + ((r0 << own.shift) + ((uint64_t)own.own_val << own.lane_bits)) * (uint64_t)cols;
                CUDA_TRY(cudaMemcpy2DAsync(stage.ptr, leaf_bytes, from, leaf_bytes << own.shift, leaf_bytes,
                                           (size_t)(count >> own.lane_bits), cudaMemcpyDefault, c->stream));
            }
            CUDA_TRY(scatter(stage.ptr, r0, count));
        }
    }
    CUDA_TRY(cudaStreamSynchronize(c->stream));     /* before the stage is freed */
    return B200DPF_OK;
}

/* Write the rows of placement P from `src`, the caller's table of P.n rows, padded to 64-byte rows */
int fill_table(b200dpf_ctx *c, const int32_t *src, const RowPlacement &P, DeviceBuffer<int32_t> *keep = nullptr)
{
    return write_rows(c, src, P.n, c->entry_size, P, [&](const int32_t *chunk, uint64_t first, uint64_t count) {
        return launch_fill_table(chunk, first, count, c->d_table.ptr, P, c->entry_size, c->entry_pad, c->sm_count, c->stream);
    }, keep);
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

/* The CPU entry points of every kind of key; `name` is the entry point's, without "b200dpf_", in messages. */

/* one key pair from the ChaCha20 DRBG: b200dpf_gen_secure for standard keys */
int gen_drbg_one(int kind, int64_t alpha, int64_t n, const uint8_t *seed, int prf, int32_t *key_a, int32_t *key_b)
{
    if (kind == host::KIND_STANDARD) return host::gen_secure(alpha, n, seed, prf, key_a, key_b);
    return host::gen_leaves(kind, alpha, n, seed, prf, key_a, key_b);
}

int gen_drbg(int kind, const char *name, int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf,
             int32_t *key_a, int32_t *key_b)
{
    const host::KindInfo &k = host::kKinds[kind];
    if (!key_a || !key_b) return fail(B200DPF_EINVAL, "null key buffer");
    if (!seed || seed_len < 44) return fail(B200DPF_EINVAL, "%s needs at least 44 bytes of seed (got %zu)", name, seed_len);
    if (gen_drbg_one(kind, alpha, n, seed, prf, key_a, key_b) != 0)
        return fail(B200DPF_EINVAL, "%s: need power-of-two n in [%lld, 2^%d], 0 <= alpha < n, valid prf (alpha=%lld n=%lld prf=%d)",
                    name, (long long)k.n_min, ilog2(k.n_max), (long long)alpha, (long long)n, prf);
    return B200DPF_OK;
}

int gen_batch_drbg(int kind, const char *name, const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                   int nthreads, int32_t *keys_a, int32_t *keys_b)
{
    if (!alphas || !seeds44 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad %s argument", name);
    if (!gen_parallel(count, nthreads, [&](int64_t i) {
            return gen_drbg_one(kind, alphas[i], n, seeds44 + 44 * i, prf, keys_a + i * host::KEY_WORDS, keys_b + i * host::KEY_WORDS);
        }))
        return fail(B200DPF_EINVAL, "%s: invalid alpha/n/prf in batch", name);
    return B200DPF_OK;
}

/* gen_batch_drbg on a GPU (b200dpf_gen_batch_gpu, _et, _xor): host alphas and seeds, keys to host or device
 * memory; `cpu_name` is the CPU entry point of the same keys, named when there is no device */
int gen_batch_gpu_kind(int kind, const char *name, const char *cpu_name, const int64_t *alphas, const uint8_t *seeds44,
                       int64_t count, int64_t n, int prf, int device, int32_t *keys_a, int32_t *keys_b)
{
    const host::KindInfo &k = host::kKinds[kind];
    if (!alphas || !seeds44 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad %s argument", name);
    if (n < k.n_min || n > k.n_max || (n & (n - 1)) != 0)
        return fail(B200DPF_EINVAL, "n=%lld must be a power of two in [%lld, 2^%d]", (long long)n, (long long)k.n_min, ilog2(k.n_max));
    if (prf < B200DPF_PRF_DUMMY || prf > B200DPF_PRF_AES128) return fail(B200DPF_EINVAL, "unknown prf id %d", prf);
    for (int64_t i = 0; i < count; i++)
        if (alphas[i] < 0 || alphas[i] >= n) return fail(B200DPF_EINVAL, "%s: alpha[%lld]=%lld out of range", name, (long long)i, (long long)alphas[i]);
    if (count == 0) return B200DPF_OK;
    std::optional<DeviceGuard> guard;
    char hint[64];
    snprintf(hint, sizeof hint, "use b200dpf_%s on the CPU", cpu_name);
    int rc = open_device(device, hint, &guard);
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
    KeygenParams p{};
    p.alphas = d_alphas.ptr;
    p.seeds44 = d_seeds.ptr;
    p.count = count;
    p.depth = ilog2(n) - k.lane_bits;
    p.lane_bits = k.lane_bits;
    p.te0 = d_te0.ptr;
    p.out_a = d_a.ptr;
    p.out_b = d_b.ptr;
    if (e == cudaSuccess) e = launch_keygen(prf, k.group, p, nullptr);
    if (e == cudaSuccess) e = cudaMemcpy(keys_a, d_a.ptr, key_bytes, cudaMemcpyDefault);      /* host or device destination */
    if (e == cudaSuccess) e = cudaMemcpy(keys_b, d_b.ptr, key_bytes, cudaMemcpyDefault);
    if (e != cudaSuccess) return fail(B200DPF_ECUDA, "%s: %s", name, cudaGetErrorString(e));
    return B200DPF_OK;
}

int eval_cpu_kind(int kind, const char *name, const int32_t *key, int prf, int32_t *out)
{
    if (!key || !out) return fail(B200DPF_EINVAL, "null buffer");
    const int rc = host::eval_cpu(key, kind, prf, out);
    if (rc == -1) return fail_not_kind(kind, name);
    if (rc) return fail(B200DPF_EINVAL, "%s: unknown prf id %d", name, prf);
    return B200DPF_OK;
}

int key_pack_kind(int kind, const char *name, const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    if (!key || !out) return fail(B200DPF_EINVAL, "null buffer");
    const int depth = host::key_depth(key, kind);
    if (depth < 1 || host::key_n(key, kind) < 0) return fail_not_kind(kind, name);
    const size_t need = b200dpf_key_packed_size(depth);
    if (out_cap < need) return fail(B200DPF_EINVAL, "%s: need %zu bytes, have %zu", name, need, out_cap);
    pack_compact(key, out, depth, host::kKinds[kind].magic);
    if (written) *written = need;
    return B200DPF_OK;
}

int key_unpack_kind(int kind, const char *name, const uint8_t *in, size_t in_len, int32_t *key)
{
    const host::KindInfo &k = host::kKinds[kind];
    if (!in || !key) return fail(B200DPF_EINVAL, "null buffer");
    if (in_len < 32 || std::memcmp(in, k.magic, 4) != 0) return fail(B200DPF_EINVAL, "%s: bad header", name);
    const int depth = in[4];
    bool pad_zero = true;
    for (int i = 5; i < 16; i++) pad_zero = pad_zero && in[i] == 0;
    if (depth < 1 || depth > k.max_depth || !pad_zero || in_len != b200dpf_key_packed_size(depth))
        return fail(B200DPF_EINVAL, "%s: depth %d does not match %zu bytes", name, depth, in_len);
    std::memset(key, 0, sizeof(int32_t) * host::KEY_WORDS);
    uint8_t *kb = reinterpret_cast<uint8_t *>(key);
    kb[16 * host::SLOT_DEPTH] = (uint8_t)depth;
    kb[16 * host::SLOT_DEPTH + 4] = (uint8_t)k.lane_bits;
    std::memcpy(kb + 16 * host::SLOT_ROOT, in + 16, 16);
    for (int L = 0; L < depth; L++) {
        const uint8_t *o = in + 32 + 64 * L;
        std::memcpy(kb + 16 * (host::SLOT_CW1 + 2 * L), o, 32);
        std::memcpy(kb + 16 * (host::SLOT_CW2 + 2 * L), o + 32, 32);
    }
    const uint64_t n = (uint64_t)1 << (depth + k.lane_bits);
    std::memcpy(kb + 16 * host::SLOT_N, &n, 8);
    return B200DPF_OK;
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
    return gen_drbg(host::KIND_STANDARD, "gen_secure", alpha, n, seed, seed_len, prf, key_a, key_b);
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
    return gen_batch_drbg(host::KIND_STANDARD, "gen_batch_secure", alphas, seeds44, count, n, prf, nthreads, keys_a, keys_b);
}

int b200dpf_gen_batch_gpu(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int device,
                          int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_gpu_kind(host::KIND_STANDARD, "gen_batch_gpu", "gen_batch_secure", alphas, seeds44, count, n, prf, device,
                              keys_a, keys_b);
}

int b200dpf_eval_cpu(const int32_t *key, int prf, int32_t *out_n)
{
    return eval_cpu_kind(host::KIND_STANDARD, "eval_cpu", key, prf, out_n);
}

size_t b200dpf_key_packed_size(int depth) { return depth >= 1 && depth <= 32 ? (size_t)32 + 64u * (size_t)depth : 0; }

int b200dpf_key_pack(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    return key_pack_kind(host::KIND_STANDARD, "key_pack", key, out, out_cap, written);
}

int b200dpf_key_unpack(const uint8_t *in, size_t in_len, int32_t *key)
{
    return key_unpack_kind(host::KIND_STANDARD, "key_unpack", in, in_len, key);
}

int64_t b200dpf_key_n(const int32_t *key) { return key ? host::key_n(key, host::KIND_STANDARD) : -1; }
int b200dpf_key_depth(const int32_t *key) { return key ? host::key_depth(key, host::KIND_STANDARD) : -1; }

/* ---- early-terminated keys ---- */

int b200dpf_gen_et(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf, int32_t *key_a, int32_t *key_b)
{
    return gen_drbg(host::KIND_ET, "gen_et", alpha, n, seed, seed_len, prf, key_a, key_b);
}

int b200dpf_gen_batch_et(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int nthreads,
                         int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_drbg(host::KIND_ET, "gen_batch_et", alphas, seeds44, count, n, prf, nthreads, keys_a, keys_b);
}

int b200dpf_gen_batch_gpu_et(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int device,
                             int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_gpu_kind(host::KIND_ET, "gen_batch_gpu_et", "gen_batch_et", alphas, seeds44, count, n, prf, device, keys_a,
                              keys_b);
}

int b200dpf_eval_cpu_et(const int32_t *key, int prf, int32_t *out_n)
{
    return eval_cpu_kind(host::KIND_ET, "eval_cpu_et", key, prf, out_n);
}

int b200dpf_key_pack_et(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    return key_pack_kind(host::KIND_ET, "key_pack_et", key, out, out_cap, written);
}

int b200dpf_key_unpack_et(const uint8_t *in, size_t in_len, int32_t *key)
{
    return key_unpack_kind(host::KIND_ET, "key_unpack_et", in, in_len, key);
}

/* ---- XOR-shared keys ---- */

int b200dpf_gen_xor(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf, int32_t *key_a, int32_t *key_b)
{
    return gen_drbg(host::KIND_XOR, "gen_xor", alpha, n, seed, seed_len, prf, key_a, key_b);
}

int b200dpf_gen_batch_xor(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int nthreads,
                          int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_drbg(host::KIND_XOR, "gen_batch_xor", alphas, seeds44, count, n, prf, nthreads, keys_a, keys_b);
}

int b200dpf_gen_batch_gpu_xor(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int device,
                              int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_gpu_kind(host::KIND_XOR, "gen_batch_gpu_xor", "gen_batch_xor", alphas, seeds44, count, n, prf, device, keys_a,
                              keys_b);
}

int b200dpf_eval_cpu_xor(const int32_t *key, int prf, uint32_t *bits)
{
    return eval_cpu_kind(host::KIND_XOR, "eval_cpu_xor", key, prf, reinterpret_cast<int32_t *>(bits));
}

int b200dpf_key_pack_xor(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    return key_pack_kind(host::KIND_XOR, "key_pack_xor", key, out, out_cap, written);
}

int b200dpf_key_unpack_xor(const uint8_t *in, size_t in_len, int32_t *key)
{
    return key_unpack_kind(host::KIND_XOR, "key_unpack_xor", in, in_len, key);
}

}  // extern "C"

/* b200dpf_create, b200dpf_create_et, b200dpf_create_xor and (`trimmed`) b200dpf_create_trimmed: a context for keys
 * of `kind` */
static int create_impl(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int device, int shard_rank,
                       int shard_count, int kind, bool trimmed = false)
{
    if (!out) return fail(B200DPF_EINVAL, "null ctx out pointer");
    *out = nullptr;
    if (!table) return fail(B200DPF_EINVAL, "null table");
    if (kind < 0 || kind >= host::KIND_COUNT) return fail(B200DPF_EINVAL, "unknown key kind %d", kind);
    TableShape shape;
    int rc = table_shape(n, kind, trimmed, -1, &shape);
    if (rc) return rc;
    if (entry_size < 1 || entry_size > 4096) return fail(B200DPF_EINVAL, "entry_size=%d out of range [1,4096]", entry_size);
    if (shard_count < 1 || (shard_count & (shard_count - 1)) != 0 ||
        (!trimmed && (int64_t)shard_count > n / host::kKinds[kind].n_min) || shard_rank < 0 || shard_rank >= shard_count)
        return fail(B200DPF_EINVAL, "bad shard %d of %d for n=%lld", shard_rank, shard_count, (long long)n);

    std::optional<DeviceGuard> guard;
    std::unique_ptr<b200dpf_ctx> c;
    rc = ctx_open(device, true, &guard, &c);
    if (rc) return rc;
    c->shape = shape;
    c->kind = kind;
    c->trimmed = trimmed;
    c->entry_size = entry_size;
    /* rows padded to what one pass reads: 16, 32 or a multiple of 64 int32 */
    c->entry_pad = entry_size <= 16 ? 16 : (entry_size <= 32 ? 32 : ((entry_size + 63) & ~63));
    c->shard_rank = shard_rank;
    c->shard_count = shard_count;
    c->shard_bits = ilog2(shard_count);
    c->place = place_of(shape, c->lane_bits(), trimmed, shard_rank, c->shard_bits);

    const size_t table_bytes = (size_t)c->rows_local() * (size_t)c->entry_pad * sizeof(int32_t);
    rc = c->d_table.reserve(table_bytes);
    if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_table.ptr, 0, table_bytes, c->stream));
    rc = fill_table(c.get(), table, c->place);
    if (rc) return rc;

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
        smem_layout(c.get(), prf, std::min(nv0, kKindOps[kind].max_nv), kKindOps[kind].mode_fused, &tmp);
        smem_layout(c.get(), prf, 4, MODE_FRONTIER, &tmp);
    }
    *out = c.release();
    return B200DPF_OK;
}

extern "C" {

int b200dpf_create(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int device,
                   int shard_rank, int shard_count)
{
    return create_impl(out, table, n, entry_size, device, shard_rank, shard_count, host::KIND_STANDARD);
}

int b200dpf_create_et(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int device,
                      int shard_rank, int shard_count)
{
    return create_impl(out, table, n, entry_size, device, shard_rank, shard_count, host::KIND_ET);
}

int b200dpf_create_xor(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int device,
                       int shard_rank, int shard_count)
{
    return create_impl(out, table, n, entry_size, device, shard_rank, shard_count, host::KIND_XOR);
}

int b200dpf_create_trimmed(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int device, int kind)
{
    return create_impl(out, table, n, entry_size, device, 0, 1, kind, true);
}

int b200dpf_ctx_rows_per_leaf(const b200dpf_ctx *c) { return c ? 1 << c->lane_bits() : -1; }

int b200dpf_ctx_trimmed(const b200dpf_ctx *c) { return c ? (c->trimmed ? 1 : 0) : -1; }

int64_t b200dpf_trimmed_domain(int64_t n, int kind) { return trim_args_ok(n, kind) ? trimmed_domain_of(n, kind) : -1; }

int64_t b200dpf_trimmed_alpha(int64_t row, int64_t n, int kind)
{
    return trim_args_ok(n, kind) && row >= 0 && row < n ? trimmed_alpha_of(row, n, kind) : -1;
}

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
        if ((rc = check_key(c, c->shape, keys + b * host::KEY_WORDS, b, -1))) return rc;
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
    const size_t stride = b200dpf_key_packed_size(c->shape.depth);
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
            if (validate && (rc = check_key(c, c->shape, keys[b], b, -1))) return rc;
            pack_compact(keys[b], stage + (size_t)b * stride, c->shape.depth, host::kKinds[c->kind].magic);
        }
        if (!c->multi)
            CUDA_TRY(cudaMemcpyAsync(reinterpret_cast<uint8_t *>(c->d_keys.ptr) + (size_t)b0 * stride, stage + (size_t)b0 * stride,
                                     (size_t)(b1 - b0) * stride, cudaMemcpyHostToDevice, c->stream));
    }
    if (c->multi) return multi_eval_host(c, stage, stride, compact_layout(c->shape.depth), nkeys, prf, out);
    return eval_tail(c, compact_layout(c->shape.depth), nkeys, prf, out);
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
    const size_t stride = b200dpf_key_packed_size(c->shape.depth);
    for (int64_t b = 0; b < nkeys; b++) {
        const uint8_t *k = packed + (size_t)b * stride;
        if (std::memcmp(k, host::kKinds[c->kind].magic, 4) != 0 || k[4] != (uint8_t)c->shape.depth)
            return fail(B200DPF_EINVAL, "packed key %lld: bad header or depth %d, table has depth %d (n=%lld)", (long long)b,
                        (int)k[4], c->shape.depth, (long long)c->shape.n);
    }
    if (c->multi) return multi_eval_host(c, packed, stride, compact_layout(c->shape.depth), nkeys, prf, out);
    return eval_host(c, packed, (size_t)nkeys * stride, compact_layout(c->shape.depth), nkeys, prf, out);
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
    return run_pipeline(c, keys_dev, reference_layout(), nkeys, prf, MODE_FUSED, out_dev,
                        reinterpret_cast<cudaStream_t>(cuda_stream));
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
    if (c->trimmed) return fail(B200DPF_ESTATE, "expand needs a context that is not trimmed");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    return run_pipeline(c, keys_dev, reference_layout(), nkeys, prf, MODE_EXPAND, shares_dev,
                        reinterpret_cast<cudaStream_t>(cuda_stream));
}

int64_t b200dpf_ctx_n(const b200dpf_ctx *c) { return c ? c->shape.n : -1; }
int b200dpf_ctx_entry_size(const b200dpf_ctx *c) { return c ? c->entry_size : -1; }
int b200dpf_ctx_device(const b200dpf_ctx *c) { return c ? c->device : -1; }
int b200dpf_ctx_last_launches(const b200dpf_ctx *c)
{
    if (!c) return -1;
    return c->multi ? multi_last_launches(c) : c->last_launches;
}

/* The plans a grouped context keeps were made under its old options */
static void options_changed(b200dpf_ctx *c)
{
    if (c->bins) {
        c->bins->cached_valid = false;
        c->bins->device_planned.valid = false;
    }
}

int b200dpf_ctx_set_subtree_log2(b200dpf_ctx *c, int s)
{
    if (!c || s < 0 || s > 16) return fail(B200DPF_EINVAL, "subtree log2 out of range");
    c->knobs.subtree_log2 = s;
    options_changed(c);
    return B200DPF_OK;
}

int b200dpf_ctx_set_option(b200dpf_ctx *c, const char *name, int value)
{
    if (!c || !name) return fail(B200DPF_EINVAL, "null argument");
    if (c->multi) return multi_set_option(c, name, value);
    for (const KnobInfo &k : kKnobs)
        if (std::strcmp(k.name, name) == 0) {
            if (value < k.lo || value > k.hi) return fail(B200DPF_EINVAL, "option %s=%d out of range [%d,%d]", name, value, k.lo, k.hi);
            c->knobs.*k.field = value;
            options_changed(c);
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
    root->shape = M->sub[0]->shape;     /* the whole table's */
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
/* The context every grouped create function starts from: bins of n[g] rows for keys of `kind`, their shapes,
 * placements and per-bin tables on the device (enqueued on the context's stream), and a zeroed device table, current
 * while `guard` lives.  `tables` (null: not checked) are the bins' sources.  n and the row offsets count rows, the
 * depths (per bin and the context's deepest) leaves. */
static int group_open(const int32_t *const *tables, const int64_t *n, int nbins, int entry_size, int device, int kind,
                      bool trimmed, std::optional<DeviceGuard> *guard, std::unique_ptr<b200dpf_ctx> *out)
{
    if (!n || nbins < 1 || nbins > (1 << 20)) return fail(B200DPF_EINVAL, "bad bin list (nbins=%d)", nbins);
    if (entry_size < 1 || entry_size > 4096) return fail(B200DPF_EINVAL, "entry_size=%d out of range [1,4096]", entry_size);
    if (kind < 0 || kind >= host::KIND_COUNT) return fail(B200DPF_EINVAL, "unknown key kind %d", kind);
    std::vector<TableShape> shape((size_t)nbins);
    TableShape all{};                   /* the context's (b200dpf_ctx::shape) */
    for (int g = 0; g < nbins; g++) {
        if (tables && !tables[g]) return fail(B200DPF_EINVAL, "bin %d: null table", g);
        TableShape &t = shape[(size_t)g];
        const int rc = table_shape(n[g], kind, trimmed, g, &t);
        if (rc) return rc;
        t.first = (uint64_t)all.rows;
        all.n = std::max(all.n, t.n);
        all.depth = std::max(all.depth, t.depth);   /* the launch plan (shared memory for correction words) is sized by it */
        all.rows += t.rows;
    }
    std::unique_ptr<b200dpf_ctx> &c = *out;
    int rc = ctx_open(device, false, guard, &c);     /* grouped contexts keep the default knobs */
    if (rc) return rc;
    c->bins.reset(new (std::nothrow) GroupBins());
    if (!c->bins) return fail(B200DPF_ENOMEM, "out of host memory");
    GroupBins *B = c->bins.get();
    B->shape = std::move(shape);
    c->shape = all;
    c->kind = kind;
    c->trimmed = trimmed;
    c->entry_size = entry_size;
    c->entry_pad = (entry_size + 15) & ~15;       /* 16 columns per pass */
    CUDA_TRY(cudaMemsetAsync(c->d_gridbar.ptr, 0, sizeof(uint32_t), c->stream));
    if (!c->coop_ok) return fail(B200DPF_ECUDA, "grouped evaluation needs cooperative launch support");
    const size_t table_bytes = (size_t)all.rows * (size_t)c->entry_pad * sizeof(int32_t);
    rc = c->d_table.reserve(table_bytes);
    if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_table.ptr, 0, table_bytes, c->stream));
    std::vector<RowPlacement> place;
    std::vector<uint2> query_bins;
    std::vector<GroupBinInfo> info;
    for (int g = 0; g < nbins; g++) {
        /* each bin in its own breadth-first leaf order (bit reversal over ITS depth), or trimmed in row order */
        const TableShape &t = B->shape[(size_t)g];
        place.push_back(place_of(t, c->lane_bits(), trimmed, 0, 0));
        info.push_back(GroupBinInfo{t.first * (uint64_t)(c->entry_pad / 4), (uint32_t)t.rows, t.depth, t.room, 0u});
        query_bins.push_back(make_uint2((uint32_t)B->query_v, (uint32_t)t.depth));
        B->query_v += b200dpf_key_packed_size(t.depth) / 16u;
    }
    const size_t bins_bytes = (size_t)nbins * sizeof(uint2), place_bytes = (size_t)nbins * sizeof(RowPlacement);
    const size_t info_bytes = (size_t)nbins * sizeof(GroupBinInfo);
    rc = B->d_place.reserve(place_bytes);
    if (!rc) rc = B->d_bins.reserve(bins_bytes);
    if (!rc) rc = B->d_bin_info.reserve(info_bytes);
    if (!rc) rc = B->d_te0.reserve(256 * sizeof(uint32_t));
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(B->d_place.ptr, place.data(), place_bytes, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaMemcpyAsync(B->d_bins.ptr, query_bins.data(), bins_bytes, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaMemcpyAsync(B->d_bin_info.ptr, info.data(), info_bytes, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaMemcpyAsync(B->d_te0.ptr, host::aes_te0(), 256 * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    /* the staging above is pageable: every copy has been taken from it when cudaMemcpyAsync returns */
    return B200DPF_OK;
}

/* b200dpf_group_create, _et, _xor and _trimmed: a grouped context for keys of `kind`, each bin uploaded from its
 * caller's table. */
static int group_create_impl(b200dpf_ctx **out, const int32_t *const *tables, const int64_t *n, int nbins, int entry_size,
                             int device, int kind, bool trimmed = false)
{
    if (!out) return fail(B200DPF_EINVAL, "null ctx out pointer");
    *out = nullptr;
    if (!tables) return fail(B200DPF_EINVAL, "bad bin list (nbins=%d)", nbins);
    std::optional<DeviceGuard> guard;
    std::unique_ptr<b200dpf_ctx> c;
    int rc = group_open(tables, n, nbins, entry_size, device, kind, trimmed, &guard, &c);
    if (rc) return rc;
    DeviceBuffer<int32_t> stage;
    for (int g = 0; g < nbins; g++) {
        rc = fill_table(c.get(), tables[g], place_of(c->bins->shape[(size_t)g], c->lane_bits(), trimmed, 0, 0), &stage);
        if (rc) return rc;
    }
    *out = c.release();
    return B200DPF_OK;
}

int b200dpf_group_create(b200dpf_ctx **out, const int32_t *const *tables, const int64_t *n, int nbins, int entry_size,
                         int device)
{
    return group_create_impl(out, tables, n, nbins, entry_size, device, host::KIND_STANDARD);
}

int b200dpf_group_create_et(b200dpf_ctx **out, const int32_t *const *tables, const int64_t *n, int nbins, int entry_size,
                            int device)
{
    return group_create_impl(out, tables, n, nbins, entry_size, device, host::KIND_ET);
}

int b200dpf_group_create_xor(b200dpf_ctx **out, const int32_t *const *tables, const int64_t *n, int nbins, int entry_size,
                             int device)
{
    return group_create_impl(out, tables, n, nbins, entry_size, device, host::KIND_XOR);
}

int b200dpf_group_create_trimmed(b200dpf_ctx **out, const int32_t *const *tables, const int64_t *n, int nbins, int entry_size,
                                 int device, int kind)
{
    return group_create_impl(out, tables, n, nbins, entry_size, device, kind, true);
}

/* The argument checks every grouped entry point makes first, in this order: the context, its buffers (`bufs`: none
 * is null), the count (nkeys keys or, with `queries`, nqueries queries of one key per bin), the prf and the
 * key_format (the evaluations of a key list take wire keys). */
static int check_group_args(const b200dpf_ctx *c, bool bufs, int64_t count, bool queries, int prf, int key_format)
{
    if (!c || !c->bins) return fail(B200DPF_ESTATE, "not a grouped context (b200dpf_group_create)");
    if (!bufs) return fail(B200DPF_EINVAL, "null buffer");
    const int per_query = queries ? (int)c->bins->shape.size() : 1;
    if (count < 1 || count > ((int64_t)1 << 24) / per_query)
        return queries ? fail(B200DPF_EINVAL, "nqueries=%lld out of range: 1 <= nqueries * nbins (%d) <= 2^24",
                              (long long)count, per_query)
                       : fail(B200DPF_EINVAL, "nkeys=%lld out of range", (long long)count);
    if (prf < B200DPF_PRF_DUMMY || prf > B200DPF_PRF_AES128) return fail(B200DPF_EINVAL, "unknown prf id %d", prf);
    if (key_format != B200DPF_KEYS_WIRE && key_format != B200DPF_KEYS_COMPACT)
        return fail(B200DPF_EINVAL, "unknown key_format %d", key_format);
    return B200DPF_OK;
}

/* The counting sort of the keys by bin (a key group must not mix bins), up to its positions: the keys of bin g go to
 * sorted positions count[g] .. count[g + 1], in the caller's order (GroupLaunch::plan places them).  Every bin id is
 * checked and, given host `keys`, every key, key by key. */
static int group_count(const b200dpf_ctx *c, const int32_t *keys, const int32_t *bins, int64_t nkeys,
                       std::vector<int64_t> *count_out)
{
    const GroupBins *B = c->bins.get();
    const int nbins = (int)B->shape.size();
    std::vector<int64_t> &count = *count_out;
    count.assign((size_t)nbins + 1, 0);
    for (int64_t b = 0; b < nkeys; b++) {
        const int g = bins[b];
        if (g < 0 || g >= nbins) return fail(B200DPF_EINVAL, "key %lld: bin %d out of range [0,%d)", (long long)b, g, nbins);
        if (keys) {
            const int rc = check_key(c, B->shape[(size_t)g], keys + b * host::KEY_WORDS, b, g);
            if (rc) return rc;
        }
        count[(size_t)g + 1]++;
    }
    for (int g = 0; g < nbins; g++) count[(size_t)g + 1] += count[(size_t)g];
    return B200DPF_OK;
}

/* Plan an evaluation of keys sorted by bin (bin g at positions count[g] .. count[g + 1]) into the staging: the key
 * groups' descriptors, for modes that draw work units their units, and the order list.  The keys come in the
 * caller's order with key b in bin bins[b] (null: nkeys / nbins queries of one key per bin, key g of query q at
 * caller's index q * nbins + g, so the sort is a fixed transpose).  The device lists grow to match. */
int GroupLaunch::plan(b200dpf_ctx *c, int prf, const std::vector<int64_t> &count, const int32_t *bins)
{
    const GroupBins *B = c->bins.get();
    const int nbins = (int)B->shape.size();
    if (!ev_staged) CUDA_TRY(cudaEventCreateWithFlags(&ev_staged, cudaEventDisableTiming));
    if (staged_pending) {             /* the previous uploads read the staging rewritten below */
        CUDA_TRY(cudaEventSynchronize(ev_staged));
        staged_pending = false;
    }
    int rc = plan_group_eval(c, prf, count, &P);
    if (rc) return rc;
    nkeys = count.back();
    const int64_t ngroups = P.key_groups;
    const size_t descs_bytes = std::max<size_t>((size_t)ngroups, 1024) * sizeof(GroupDesc);
    const size_t order_bytes = std::max<size_t>((size_t)nkeys, 1024) * sizeof(uint2);
    rc = h_descs.reserve(descs_bytes);
    if (!rc) rc = d_descs.reserve(descs_bytes);
    if (!rc) rc = h_order.reserve(order_bytes);
    if (!rc) rc = d_order.reserve(order_bytes);
    if (rc) return rc;
    {
        int64_t gi = 0;
        for (int g = 0; g < nbins; g++) {
            const TableShape &t = B->shape[(size_t)g];
            const int s = group_s(P, *B, g);
            for (int64_t k = count[(size_t)g]; k < count[(size_t)g + 1]; k += 32, gi++) {
                GroupDesc &d = h_descs.ptr[gi];
                d.key_first = (uint32_t)k;
                d.nkeys = (uint32_t)std::min<int64_t>(32, count[(size_t)g + 1] - k);
                d.depth = t.depth;
                d.s = s;
                d.nsub = (uint32_t)(t.rows >> (s + c->lane_bits()));   /* 2^(depth - s) unless trimmed */
                d.pad = 0;
                d.table_off_v = t.first * (uint64_t)(c->entry_pad / 4);
            }
        }
    }
    /* modes that draw work units: every key group's items, in group-major order, cut evenly into units of
     * at most one item per warp of a block.  A unit's items run side by side, so a launch takes about
     * (units per block) unit times: whole-block units unless the launch holds fewer items than the grid
     * has warps, and then about items / blocks per unit, so that every block has work.  A key group with
     * fewer items than its unit size leaves the rest of its unit's warps idle. */
    nunits = 0;
    if (mode_traits(P.mode).units) {
        int64_t items = 0;
        for (int64_t gi = 0; gi < ngroups; gi++) items += h_descs.ptr[gi].nsub;
        const int64_t per_unit = std::clamp<int64_t>((items + P.L.grid - 1) / P.L.grid, 1, P.L.threads / 32);
        for (int64_t gi = 0; gi < ngroups; gi++) nunits += (h_descs.ptr[gi].nsub + per_unit - 1) / per_unit;
        const size_t units_bytes = std::max<size_t>((size_t)nunits, 1024) * sizeof(WorkUnit);
        rc = h_units.reserve(units_bytes);
        if (!rc) rc = d_units.reserve(units_bytes);
        if (rc) return rc;
        WorkUnit *w = h_units.ptr;
        for (int64_t gi = 0; gi < ngroups; gi++) {
            const uint64_t nsub = h_descs.ptr[gi].nsub;
            const uint64_t parts = (nsub + (uint64_t)per_unit - 1) / (uint64_t)per_unit;
            for (uint64_t j = 0; j < parts; j++) {
                const uint64_t first = nsub * j / parts, end = nsub * (j + 1) / parts;
                *w++ = WorkUnit{(uint32_t)gi, (uint32_t)first, (uint32_t)(end - first), 0u};
            }
        }
    }
    if (bins) {
        std::vector<int64_t> next(count.begin(), count.end() - 1);
        for (int64_t b = 0; b < nkeys; b++)
            h_order.ptr[next[(size_t)bins[b]]++] = make_uint2((uint32_t)b, (uint32_t)B->shape[(size_t)bins[b]].depth);
    } else {
        const int64_t nq = nkeys / nbins;
        for (int g = 0; g < nbins; g++)
            for (int64_t q = 0; q < nq; q++)
                h_order.ptr[g * nq + q] = make_uint2((uint32_t)(q * nbins + g), (uint32_t)B->shape[(size_t)g].depth);
    }
    return B200DPF_OK;
}

/* Upload the lists of the last plan on `stream` (the order list only if `order`), then record ev_staged. */
int GroupLaunch::upload(cudaStream_t stream, bool order)
{
    CUDA_TRY(cudaMemcpyAsync(d_descs.ptr, h_descs.ptr, (size_t)P.key_groups * sizeof(GroupDesc), cudaMemcpyHostToDevice, stream));
    if (mode_traits(P.mode).units)
        CUDA_TRY(cudaMemcpyAsync(d_units.ptr, h_units.ptr, (size_t)nunits * sizeof(WorkUnit), cudaMemcpyHostToDevice, stream));
    if (order) CUDA_TRY(cudaMemcpyAsync(d_order.ptr, h_order.ptr, (size_t)nkeys * sizeof(uint2), cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaEventRecord(ev_staged, stream));
    staged_pending = true;
    return B200DPF_OK;
}

/* The evaluation by plan P of nkeys keys, sorted by bin and compact in d_keys, into d_out in sorted order: the key
 * groups' descriptors, the work units (nunits of them, or a bound of them when `counts` holds their counts) */
static int group_launch_lists(b200dpf_ctx *c, const EvalPlan &P, int64_t nkeys, const GroupDesc *descs, const WorkUnit *units,
                              uint32_t nunits, const uint32_t *counts, int prf, cudaStream_t stream)
{
    const EvalJob J{c->d_keys.ptr, compact_layout(c->shape.depth), nkeys, prf, MODE_FUSED, c->d_out.ptr, stream, true, false,
                    descs, units, nunits, true, counts};
    return launch_plan(c, J, P);
}

static int group_launch(b200dpf_ctx *c, const GroupLaunch &L, int prf, cudaStream_t stream)
{
    return group_launch_lists(c, L.P, L.nkeys, L.d_descs.ptr, L.d_units.ptr, (uint32_t)L.nunits, nullptr, prf, stream);
}

int b200dpf_group_eval(b200dpf_ctx *c, const int32_t *keys, const int32_t *bins, int64_t nkeys, int prf, int32_t *out)
{
    int rc = check_group_args(c, keys && bins && out, nkeys, false, prf, B200DPF_KEYS_WIRE);
    if (rc) return rc;
    std::vector<int64_t> count;
    rc = group_count(c, keys, bins, nkeys, &count);
    if (rc) return rc;
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    GroupLaunch &L = c->bins->once;
    rc = L.plan(c, prf, count, bins);
    if (rc) return rc;
    /* keys travel in the compact layout, one stride for all bins (that of the deepest): a key for a
     * 2^10-entry bin has 672 live bytes of its 2096 (early-terminated: 544) */
    const KeyLayout kl = compact_layout(c->shape.depth);
    const char *magic = host::kKinds[c->kind].magic;
    const size_t stride = (size_t)kl.stride_v * 16u;
    const size_t key_bytes = (size_t)nkeys * stride;
    rc = reserve_host_keys(c, key_bytes);
    if (rc) return rc;
    const uint2 *order = L.h_order.ptr;
    {
        uint8_t *stage = reinterpret_cast<uint8_t *>(c->h_keys.ptr);
        auto pack_range = [&](int64_t p0, int64_t p1) {
            for (int64_t pos = p0; pos < p1; pos++)
                pack_compact(keys + (size_t)order[pos].x * host::KEY_WORDS, stage + (size_t)pos * stride, (int)order[pos].y, magic);
        };
        const int nthr = (int)std::min<int64_t>(std::min<int64_t>(8, std::max(1u, std::thread::hardware_concurrency())), nkeys / 2048 + 1);
        std::vector<std::thread> pool;
        for (int t = 1; t < nthr; t++) pool.emplace_back(pack_range, nkeys * t / nthr, nkeys * (t + 1) / nthr);
        pack_range(0, nkeys / nthr);
        for (auto &th : pool) th.join();
    }
    const size_t out_elems = (size_t)nkeys * c->entry_size;
    rc = reserve_device_io(c, key_bytes, out_elems);
    if (!rc) rc = reserve_host_out(c, out_elems);
    if (!rc) rc = wait_last(c, c->stream);
    if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->d_keys.ptr, c->h_keys.ptr, key_bytes, cudaMemcpyHostToDevice, c->stream));
    rc = L.upload(c->stream, false);
    if (!rc) rc = group_launch(c, L, prf, c->stream);
    if (!rc) rc = download_out(c, c->h_out.ptr, true, out_elems);
    if (rc) return rc;
    for (int64_t pos = 0; pos < nkeys; pos++)       /* back to the caller's order */
        std::memcpy(out + (size_t)order[pos].x * c->entry_size, c->h_out.ptr + pos * c->entry_size, sizeof(int32_t) * (size_t)c->entry_size);
    return B200DPF_OK;
}

/* The end of both device-resident grouped evaluations, on `stream` and after the context's last operation: launch
 * L's lists go up if its caller just planned it (`upload`), a gather puts the caller's keys into bin order in
 * d_keys (wire keys through the order list, compact queries through the per-bin table), the evaluation runs, and
 * a scatter puts its results back into the caller's order in out_dev. */
static int group_enqueue(b200dpf_ctx *c, GroupLaunch &L, bool upload, const void *keys_dev, int key_format, int prf,
                         void *out_dev, cudaStream_t stream)
{
    const GroupBins *B = c->bins.get();
    const KeyLayout kl = compact_layout(c->shape.depth);
    int rc = reserve_device_io(c, (size_t)L.nkeys * kl.stride_v * 16u, (size_t)L.nkeys * c->entry_size);
    if (!rc) rc = wait_last(c, stream);
    if (!rc && upload) rc = L.upload(stream, true);
    if (rc) return rc;
    uint32_t magic = 0;
    std::memcpy(&magic, host::kKinds[c->kind].magic, 4);
    if (key_format == B200DPF_KEYS_WIRE)
        CUDA_TRY(launch_group_gather(keys_dev, L.d_order.ptr, L.nkeys, magic, kl.stride_v, c->d_keys.ptr, stream));
    else
        CUDA_TRY(launch_group_gather_queries(keys_dev, B->d_bins.ptr, L.nkeys, (uint32_t)(L.nkeys / (int64_t)B->shape.size()),
                                             B->query_v, magic, kl.stride_v, c->d_keys.ptr, stream));
    rc = group_launch(c, L, prf, stream);
    if (rc) return rc;
    CUDA_TRY(launch_group_scatter(c->d_out.ptr, L.d_order.ptr, L.nkeys, c->entry_size, out_dev, stream));
    return mark_last(c, stream);
}

/* The same evaluation from device keys into device results, enqueued on the caller's stream: the host sorts
 * and plans from the bins alone, a gather kernel packs the keys into bin order (what pack_compact does on the
 * host path), the evaluation is that of b200dpf_group_eval, and a scatter kernel puts the results back into
 * the caller's order.  The only host wait is for the previous call's uploads from the pinned staging. */
int b200dpf_group_eval_device(b200dpf_ctx *c, const void *keys_dev, const int32_t *bins, int64_t nkeys, int prf,
                              void *out_dev, void *cuda_stream)
{
    int rc = check_group_args(c, keys_dev && bins && out_dev, nkeys, false, prf, B200DPF_KEYS_WIRE);
    if (rc) return rc;
    if ((reinterpret_cast<uintptr_t>(keys_dev) & 15u) != 0 || (reinterpret_cast<uintptr_t>(out_dev) & 3u) != 0)
        return fail(B200DPF_EINVAL, "keys_dev must be 16-byte aligned and out_dev 4-byte aligned");
    std::vector<int64_t> count;
    rc = group_count(c, nullptr, bins, nkeys, &count);
    if (rc) return rc;
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    GroupLaunch &L = c->bins->once;
    rc = L.plan(c, prf, count, bins);
    return rc ? rc : group_enqueue(c, L, true, keys_dev, B200DPF_KEYS_WIRE, prf, out_dev, reinterpret_cast<cudaStream_t>(cuda_stream));
}

/* The same evaluation with the bins in device memory too: the host half of the plan (plan_group_device) is kept per
 * (nkeys, prf, options), and a call enqueues the device half (launch_group_plan: histogram, sort, plan, lists), the
 * gather, the evaluation in the mode whose counts are on the device, and the scatter.  Keys whose bin is out of
 * range sort to a tail no key group covers; the launch clears d_out, so the scatter gives them zero rows. */
int b200dpf_group_eval_device_bins(b200dpf_ctx *c, const void *keys_dev, const int32_t *bins_dev, int64_t nkeys, int prf,
                                   void *out_dev, int64_t *bad_dev, void *cuda_stream)
{
    int rc = check_group_args(c, keys_dev && bins_dev && out_dev, nkeys, false, prf, B200DPF_KEYS_WIRE);
    if (rc) return rc;
    if ((reinterpret_cast<uintptr_t>(keys_dev) & 15u) != 0 || (reinterpret_cast<uintptr_t>(out_dev) & 3u) != 0)
        return fail(B200DPF_EINVAL, "keys_dev must be 16-byte aligned and out_dev 4-byte aligned");
    if ((reinterpret_cast<uintptr_t>(bins_dev) & 3u) != 0 || (reinterpret_cast<uintptr_t>(bad_dev) & 7u) != 0)
        return fail(B200DPF_EINVAL, "bins_dev must be 4-byte aligned and bad_dev 8-byte aligned");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    const cudaStream_t stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    DevicePlanned &D = c->bins->device_planned;
    if (!D.valid || D.nkeys != nkeys || D.prf != prf) rc = plan_group_device(c, prf, nkeys, &D);
    const KeyLayout kl = compact_layout(c->shape.depth);
    if (!rc) rc = reserve_device_io(c, (size_t)nkeys * kl.stride_v * 16u, (size_t)nkeys * c->entry_size);
    if (!rc) rc = wait_last(c, stream);
    if (rc) return rc;
    GroupPlanParams gp = D.gp;
    gp.bins = bins_dev;
    gp.bad = bad_dev;
    CUDA_TRY(launch_group_plan(gp, c->sm_count, stream));
    uint32_t magic = 0;
    std::memcpy(&magic, host::kKinds[c->kind].magic, 4);
    CUDA_TRY(launch_group_gather(keys_dev, D.d_order.ptr, nkeys, magic, kl.stride_v, c->d_keys.ptr, stream));
    rc = group_launch_lists(c, D.P, nkeys, D.d_descs.ptr, D.d_units.ptr, (uint32_t)D.units_bound, D.d_counts.ptr, prf, stream);
    if (rc) return rc;
    CUDA_TRY(launch_group_scatter(c->d_out.ptr, D.d_order.ptr, nkeys, c->entry_size, out_dev, stream));
    return mark_last(c, stream);
}

/* The lists of a grouped context's last plan, for tests: which = 0, those b200dpf_group_eval_device_bins made on the
 * device (read after the context's last operation); which = 1, those b200dpf_group_eval or _eval_device made on the
 * host.  counts = (key groups, work units, keys, keys out of range); up to the caps of entries are copied. */
int b200dpf_group_plan_lists(b200dpf_ctx *c, int which, int64_t *counts, void *descs, int64_t descs_cap, void *units,
                             int64_t units_cap, void *order, int64_t order_cap)
{
    if (!c || !c->bins) return fail(B200DPF_ESTATE, "not a grouped context (b200dpf_group_create)");
    if (!counts || !descs || !units || !order || which < 0 || which > 1 || descs_cap < 0 || units_cap < 0 || order_cap < 0)
        return fail(B200DPF_EINVAL, "bad arguments");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    GroupBins *B = c->bins.get();
    if (which == 0) {
        const DevicePlanned &D = B->device_planned;
        if (!D.valid) return fail(B200DPF_ESTATE, "no b200dpf_group_eval_device_bins call to read");
        if (c->has_last) CUDA_TRY(cudaEventSynchronize(c->ev_done));
        uint32_t n[4];
        CUDA_TRY(cudaMemcpy(n, D.d_counts.ptr, sizeof n, cudaMemcpyDeviceToHost));
        counts[0] = n[0]; counts[1] = n[1]; counts[2] = D.nkeys; counts[3] = n[2];
        if (std::min<int64_t>(n[0], descs_cap) > 0)
            CUDA_TRY(cudaMemcpy(descs, D.d_descs.ptr, (size_t)std::min<int64_t>(n[0], descs_cap) * sizeof(GroupDesc), cudaMemcpyDeviceToHost));
        if (std::min<int64_t>(n[1], units_cap) > 0)
            CUDA_TRY(cudaMemcpy(units, D.d_units.ptr, (size_t)std::min<int64_t>(n[1], units_cap) * sizeof(WorkUnit), cudaMemcpyDeviceToHost));
        if (std::min<int64_t>(D.nkeys, order_cap) > 0)
            CUDA_TRY(cudaMemcpy(order, D.d_order.ptr, (size_t)std::min<int64_t>(D.nkeys, order_cap) * sizeof(uint2), cudaMemcpyDeviceToHost));
        return B200DPF_OK;
    }
    const GroupLaunch &L = B->once;
    if (!L.h_descs.ptr) return fail(B200DPF_ESTATE, "no b200dpf_group_eval or _eval_device call to read");
    counts[0] = L.P.key_groups; counts[1] = L.nunits; counts[2] = L.nkeys; counts[3] = 0;
    std::memcpy(descs, L.h_descs.ptr, (size_t)std::min<int64_t>(L.P.key_groups, descs_cap) * sizeof(GroupDesc));
    if (L.nunits) std::memcpy(units, L.h_units.ptr, (size_t)std::min<int64_t>(L.nunits, units_cap) * sizeof(WorkUnit));
    std::memcpy(order, L.h_order.ptr, (size_t)std::min<int64_t>(L.nkeys, order_cap) * sizeof(uint2));
    return B200DPF_OK;
}

int64_t b200dpf_group_query_bytes(const b200dpf_ctx *c)
{
    return c && c->bins ? (int64_t)c->bins->query_v * 16 : -1;
}

/* b200dpf_group_eval_device for Q queries of one key per bin: the plan, its device lists and the reordering are
 * those of the previous call when Q, the prf and the options are (GroupBins::cached), and a call then only
 * enqueues the stream wait, the gather, the evaluation and the scatter. */
int b200dpf_group_eval_queries_device(b200dpf_ctx *c, const void *keys_dev, int key_format, int64_t nqueries, int prf,
                                      void *out_dev, void *cuda_stream)
{
    int rc = check_group_args(c, keys_dev && out_dev, nqueries, true, prf, key_format);
    if (rc) return rc;
    if ((reinterpret_cast<uintptr_t>(keys_dev) & 15u) != 0 || (reinterpret_cast<uintptr_t>(out_dev) & 3u) != 0)
        return fail(B200DPF_EINVAL, "keys_dev must be 16-byte aligned and out_dev 4-byte aligned");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    GroupBins *B = c->bins.get();
    const bool replan = !B->cached_valid || B->cached_nq != nqueries || B->cached_prf != prf;
    if (replan) {
        std::vector<int64_t> count(B->shape.size() + 1);
        for (size_t g = 0; g < count.size(); g++) count[g] = (int64_t)g * nqueries;
        B->cached_valid = false;
        rc = B->cached.plan(c, prf, count, nullptr);
    }
    if (!rc) rc = group_enqueue(c, B->cached, replan, keys_dev, key_format, prf, out_dev, reinterpret_cast<cudaStream_t>(cuda_stream));
    if (!rc && replan) {
        B->cached_nq = nqueries;
        B->cached_prf = prf;
        B->cached_valid = true;
    }
    return rc;
}

/* The client's side of b200dpf_group_eval_queries_device: one keygen launch (one thread per (query, bin) pair,
 * dpf_keygen.cu) writes both servers' queries.  It reads only the per-bin tables of the context, not its tables of
 * rows, so it neither joins the one-operation-in-flight chain nor touches the cached plan. */
int b200dpf_group_gen_queries_device(b200dpf_ctx *c, const int64_t *alphas_dev, const uint8_t *seeds_dev, int64_t nqueries,
                                     int prf, int key_format, void *out_a_dev, void *out_b_dev, void *cuda_stream)
{
    const int rc = check_group_args(c, alphas_dev && seeds_dev && out_a_dev && out_b_dev, nqueries, true, prf, key_format);
    if (rc) return rc;
    if (((reinterpret_cast<uintptr_t>(out_a_dev) | reinterpret_cast<uintptr_t>(out_b_dev)) & 15u) != 0)
        return fail(B200DPF_EINVAL, "out_a_dev and out_b_dev must be 16-byte aligned");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    const GroupBins *B = c->bins.get();
    const int nbins = (int)B->shape.size();
    const host::KindInfo &k = host::kKinds[c->kind];
    KeygenParams p{};
    p.alphas = alphas_dev;
    p.seeds44 = seeds_dev;
    p.count = nqueries * nbins;
    p.lane_bits = k.lane_bits;
    p.bins = B->d_bins.ptr;
    p.bin_place = B->d_place.ptr;
    p.nq = (uint32_t)nqueries;
    p.nbins = (uint32_t)nbins;
    p.query_v = B->query_v;
    p.compact = key_format == B200DPF_KEYS_COMPACT;
    std::memcpy(&p.magic, k.magic, 4);
    p.te0 = B->d_te0.ptr;
    p.out_a = static_cast<uint4 *>(out_a_dev);
    p.out_b = static_cast<uint4 *>(out_b_dev);
    CUDA_TRY(launch_keygen(prf, k.group, p, reinterpret_cast<cudaStream_t>(cuda_stream)));
    return B200DPF_OK;
}

/* ------------------------------------------------------------------------------------------- */
/* Batch codes: any k rows of one table per query (DESIGN.md section 13).                        */
/* ------------------------------------------------------------------------------------------- */
/* The layout of an n-row table in nbins bins (BatchCodeLayout), or EINVAL */
static int batchcode_layout_of(int64_t n, int nbins, uint64_t seed, BatchCodeLayout *L)
{
    if (n < 1 || n > ((int64_t)1 << 31)) return fail(B200DPF_EINVAL, "table size n=%lld out of range [1, 2^31]", (long long)n);
    if (nbins < 1 || nbins > (1 << 20) || nbins > n)
        return fail(B200DPF_EINVAL, "nbins=%d out of range [1, min(n, 2^20)] (n=%lld)", nbins, (long long)n);
    int bits = 2;
    while (bits < 64 && ((int64_t)1 << bits) < n) bits += 2;
    *L = BatchCodeLayout{(uint64_t)n, seed, (uint32_t)nbins, bits / 2};
    if (BATCHCODE_COPIES * L->per_copy(0) > ((uint64_t)1 << 31))
        return fail(B200DPF_EINVAL, "bin 0 would hold %llu rows, more than 2^31: use more bins",
                    (unsigned long long)(BATCHCODE_COPIES * L->per_copy(0)));
    return B200DPF_OK;
}

/* The batch-code layout of a context, or ESTATE */
static int batchcode_of(const b200dpf_ctx *c, const BatchCodeLayout **L)
{
    if (!c || !c->bins || !c->bins->batch) return fail(B200DPF_ESTATE, "not a batch-code context (b200dpf_batchcode_create)");
    *L = &*c->bins->batch;
    return B200DPF_OK;
}

/* The argument checks both planners make: k wanted rows per query, nqueries queries of one key per bin */
static int check_plan_args(const BatchCodeLayout &L, bool bufs, int64_t nqueries, int k)
{
    if (!bufs) return fail(B200DPF_EINVAL, "null buffer");
    if (k < 1 || k > BATCHCODE_MAX_K) return fail(B200DPF_EINVAL, "k=%d out of range [1, %d]", k, (int)BATCHCODE_MAX_K);
    if (nqueries < 1 || nqueries > ((int64_t)1 << 24) / (int64_t)L.nbins)
        return fail(B200DPF_EINVAL, "nqueries=%lld out of range: 1 <= nqueries * nbins (%u) <= 2^24", (long long)nqueries, L.nbins);
    return B200DPF_OK;
}

int b200dpf_batchcode_create(b200dpf_ctx **out, const int32_t *table, int64_t n, int entry_size, int nbins, uint64_t layout_seed,
                             int device, int kind)
{
    if (!out) return fail(B200DPF_EINVAL, "null ctx out pointer");
    *out = nullptr;
    if (!table) return fail(B200DPF_EINVAL, "null table");
    BatchCodeLayout L;
    int rc = batchcode_layout_of(n, nbins, layout_seed, &L);
    if (rc) return rc;
    std::vector<int64_t> rows((size_t)nbins);
    for (int j = 0; j < nbins; j++) rows[(size_t)j] = (int64_t)(BATCHCODE_COPIES * L.per_copy((uint32_t)j));
    std::optional<DeviceGuard> guard;
    std::unique_ptr<b200dpf_ctx> c;
    rc = group_open(nullptr, rows.data(), nbins, entry_size, device, kind, true, &guard, &c);
    if (rc) return rc;
    /* each row to its three copies in the bins (placements already on the device) */
    rc = write_rows(c.get(), table, L.n, entry_size, RowPlacement{}, [&](const int32_t *chunk, uint64_t first, uint64_t count) {
        return launch_batchcode_scatter(chunk, first, count, L, c->bins->d_place.ptr, c->d_table.ptr, c->entry_size, c->entry_pad,
                                        c->stream);
    });
    if (rc) return rc;
    c->bins->batch = L;
    *out = c.release();
    return B200DPF_OK;
}

int b200dpf_batchcode_layout(const b200dpf_ctx *c, int64_t *n, int *nbins, uint64_t *seed)
{
    const BatchCodeLayout *L = nullptr;
    const int rc = batchcode_of(c, &L);
    if (rc) return rc;
    if (!n || !nbins || !seed) return fail(B200DPF_EINVAL, "null buffer");
    *n = (int64_t)L->n;
    *nbins = (int)L->nbins;
    *seed = L->seed;
    return B200DPF_OK;
}

int b200dpf_batchcode_locate(int64_t n, int nbins, uint64_t seed, int64_t row, int32_t *bins3, int64_t *rows3)
{
    BatchCodeLayout L;
    const int rc = batchcode_layout_of(n, nbins, seed, &L);
    if (rc) return rc;
    if (!bins3 || !rows3) return fail(B200DPF_EINVAL, "null buffer");
    if (row < 0 || row >= n) return fail(B200DPF_EINVAL, "row %lld out of range [0, %lld)", (long long)row, (long long)n);
    for (int c = 0; c < BATCHCODE_COPIES; c++) {
        uint32_t bin;
        uint64_t r;
        L.locate(c, (uint64_t)row, &bin, &r);
        bins3[c] = (int32_t)bin;
        rows3[c] = (int64_t)r;
    }
    return B200DPF_OK;
}

int b200dpf_batchcode_plan(int64_t n, int nbins, uint64_t seed, const int64_t *wanted, int64_t nqueries, int k, int64_t *alphas,
                           int32_t *slots)
{
    BatchCodeLayout L;
    int rc = batchcode_layout_of(n, nbins, seed, &L);
    if (!rc) rc = check_plan_args(L, wanted && alphas && slots, nqueries, k);
    if (rc) return rc;
    for (int64_t j = 0; j < nqueries * k; j++)
        if (wanted[j] < 0 || wanted[j] >= n)
            return fail(B200DPF_EINVAL, "query %lld: wanted row %lld out of range [0, %lld)", (long long)(j / k), (long long)wanted[j],
                        (long long)n);
    gen_parallel(nqueries, nqueries >= 64 ? 0 : 1, [&](int64_t q) {
        batchcode_plan_query(L, wanted + q * k, k, alphas + q * (int64_t)nbins, slots + q * k);
        return false;
    });
    return B200DPF_OK;
}

/* The planner of b200dpf_batchcode_plan, one thread per query, in the caller's buffers only: it neither joins the
 * context's one-operation-in-flight chain nor reads anything of the context on the device. */
int b200dpf_batchcode_plan_device(b200dpf_ctx *c, const int64_t *wanted_dev, int64_t nqueries, int k, int64_t *alphas_dev,
                                  int32_t *slots_dev, void *cuda_stream)
{
    const BatchCodeLayout *L = nullptr;
    int rc = batchcode_of(c, &L);
    if (!rc) rc = check_plan_args(*L, wanted_dev && alphas_dev && slots_dev, nqueries, k);
    if (rc) return rc;
    if (((reinterpret_cast<uintptr_t>(wanted_dev) | reinterpret_cast<uintptr_t>(alphas_dev)) & 7u) != 0 ||
        (reinterpret_cast<uintptr_t>(slots_dev) & 3u) != 0)
        return fail(B200DPF_EINVAL, "wanted_dev and alphas_dev must be 8-byte aligned and slots_dev 4-byte aligned");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    CUDA_TRY(launch_batchcode_plan(*L, wanted_dev, nqueries, k, alphas_dev, slots_dev, reinterpret_cast<cudaStream_t>(cuda_stream)));
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

/* Grow the scratch for `count` rows (staged: the inputs are copied into it) and order everything that
 * follows on `stream` after the context's previous evaluation or update: the update writes the table
 * those read, and the scratch is the previous update's. */
int update_begin(b200dpf_ctx *c, int64_t count, bool staged, bool with_bins, cudaStream_t stream, UpdateLayout *L)
{
    const uint64_t rows = (uint64_t)c->rows_local();
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
        u.bin_place = c->bins->d_place.ptr;
        u.nbins = (int)c->bins->shape.size();
    }
    u.place = c->place;
    u.rows = rows;
    u.count = count;
    u.table_rows = (uint32_t)c->rows_local();
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
        for (int64_t j = 0; j < count; j++)
            if (c->place.owns(idx[j])) {
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
        if (indices[j] < 0 || indices[j] >= c->shape.n)
            return fail(B200DPF_EINVAL, "update %lld: index %lld out of range [0, %lld)", (long long)j, (long long)indices[j],
                        (long long)c->shape.n);
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
    if (c->bins->batch)
        return fail(B200DPF_ESTATE, "batch-code context: one copy of a row cannot change alone, use b200dpf_batchcode_update_rows");
    if (c->bins->keyword)
        return fail(B200DPF_ESTATE, "keyword-PIR context: a row update could overwrite a tag, use b200dpf_kwpir_update");
    if (count > 0 && !bins) return fail(B200DPF_EINVAL, "null buffer");
    GroupBins *B = c->bins.get();
    const int nbins = (int)B->shape.size();
    for (int64_t j = 0; j < count; j++) {
        if (bins[j] < 0 || bins[j] >= nbins)
            return fail(B200DPF_EINVAL, "update %lld: bin %d out of range [0,%d)", (long long)j, bins[j], nbins);
        if (indices[j] < 0 || indices[j] >= B->shape[(size_t)bins[j]].n)
            return fail(B200DPF_EINVAL, "update %lld: index %lld out of range [0, %lld) of bin %d", (long long)j,
                        (long long)indices[j], (long long)B->shape[(size_t)bins[j]].n, bins[j]);
    }
    if (count == 0) return B200DPF_OK;
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    rc = update_host_enqueue(c, indices, bins, rows, count);
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    return B200DPF_OK;
}

/* All three copies of each row, through the grouped update path: entry j becomes entries 3j, 3j + 1, 3j + 2, one per
 * copy, so the last occurrence of a row still wins in every copy. */
int b200dpf_batchcode_update_rows(b200dpf_ctx *c, const int64_t *indices, const int32_t *rows, int64_t count)
{
    const BatchCodeLayout *L = nullptr;
    int rc = batchcode_of(c, &L);
    if (!rc) rc = check_update_args(c, indices, rows, count);
    if (rc) return rc;
    if (count > kMaxUpdateCount / BATCHCODE_COPIES)
        return fail(B200DPF_EINVAL, "update count=%lld out of range [0, (2^31 - 1) / 3]", (long long)count);
    for (int64_t j = 0; j < count; j++)
        if (indices[j] < 0 || (uint64_t)indices[j] >= L->n)
            return fail(B200DPF_EINVAL, "update %lld: index %lld out of range [0, %lld)", (long long)j, (long long)indices[j],
                        (long long)L->n);
    if (count == 0) return B200DPF_OK;
    const size_t E = (size_t)c->entry_size;
    std::vector<int32_t> bins3((size_t)count * BATCHCODE_COPIES);
    std::vector<int64_t> idx3(bins3.size());
    std::vector<int32_t> rows3(bins3.size() * E);
    for (int64_t j = 0; j < count; j++)
        for (int k = 0; k < BATCHCODE_COPIES; k++) {
            const size_t e = (size_t)j * BATCHCODE_COPIES + k;
            uint32_t bin;
            uint64_t row;
            L->locate(k, (uint64_t)indices[j], &bin, &row);
            bins3[e] = (int32_t)bin;
            idx3[e] = (int64_t)row;
            std::memcpy(rows3.data() + e * E, rows + (size_t)j * E, E * sizeof(int32_t));
        }
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    rc = update_host_enqueue(c, idx3.data(), bins3.data(), rows3.data(), (int64_t)bins3.size());
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    return B200DPF_OK;
}

/* ------------------------------------------------------------------------------------------- */
/* Keyword PIR: a value by its 64-bit keyword in one query (DESIGN.md section 14).               */
/* ------------------------------------------------------------------------------------------- */
static int kwpir_check_m(int64_t m)
{
    if (m < 1 || m > ((int64_t)1 << 31)) return fail(B200DPF_EINVAL, "m=%lld slots per table out of range [1, 2^31]", (long long)m);
    return B200DPF_OK;
}

/* The keyword-PIR layout of n items in tables of m slots (KeywordLayout), or EINVAL */
static int kwpir_layout_of(int64_t n, int value_size, int64_t m, uint64_t seed, KeywordLayout *L)
{
    if (n < 1 || n > ((int64_t)1 << 30)) return fail(B200DPF_EINVAL, "item count n=%lld out of range [1, 2^30]", (long long)n);
    if (value_size < 1 || value_size > KWPIR_MAX_VALUE)
        return fail(B200DPF_EINVAL, "value_size=%d out of range [1, %d]", value_size, (int)KWPIR_MAX_VALUE);
    if (m < (n + 2) / 3 || m > ((int64_t)1 << 31))
        return fail(B200DPF_EINVAL, "m=%lld slots per table out of range [ceil(n / 3) = %lld, 2^31]", (long long)m, (long long)((n + 2) / 3));
    *L = KeywordLayout{(uint64_t)n, (uint64_t)m, seed, value_size};
    return B200DPF_OK;
}

/* The keyword state of a context, or ESTATE */
static int kwpir_of(const b200dpf_ctx *c, const GroupBins::Keyword **K)
{
    if (!c || !c->bins || !c->bins->keyword) return fail(B200DPF_ESTATE, "not a keyword-PIR context (b200dpf_kwpir_create)");
    *K = &*c->bins->keyword;
    return B200DPF_OK;
}

static int kwpir_reserved(const uint64_t *keywords, int64_t count)
{
    for (int64_t j = 0; j < count; j++)
        if (keywords[j] == ~0ull) return fail(B200DPF_EINVAL, "keyword %lld is 2^64 - 1, which is reserved (tag 0 marks an empty slot)", (long long)j);
    return B200DPF_OK;
}

/* Refuse duplicate and reserved keywords, place every item by the rounds of the layout's rule and write the rows into
 * the bins of c (placements already on the device), then wait.  Scratch: O(n + m) device memory, freed on return. */
static int kwpir_build(b200dpf_ctx *c, const uint64_t *keywords, const int32_t *values, const KeywordLayout &L,
                       GroupBins::Keyword *K)
{
    const cudaStream_t st = c->stream;
    const uint64_t n = L.n, slots = KWPIR_TABLES * L.m;
    bool kw_on_device;
    int kw_device;
    int rc = wait_source(c, keywords, &kw_on_device, &kw_device);
    if (rc) return rc;
    DeviceBuffer<uint64_t> d_keys, d_sorted;
    DeviceBuffer<char> d_temp;
    DeviceBuffer<uint32_t> d_words;       /* [0] flags, [1] next homeless count */
    const uint64_t *keys = keywords;
    if (!kw_on_device || kw_device != c->device) {
        rc = d_keys.reserve(n * sizeof(uint64_t));
        if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(d_keys.ptr, keywords, n * sizeof(uint64_t), cudaMemcpyDefault, st));
        keys = d_keys.ptr;
    }
    size_t temp_bytes = 0;
    CUDA_TRY(kwpir_check_temp_bytes(n, &temp_bytes));
    rc = d_sorted.reserve(n * sizeof(uint64_t));
    if (!rc) rc = d_temp.reserve(std::max<size_t>(temp_bytes, 1));
    if (!rc) rc = d_words.reserve(2 * sizeof(uint32_t));
    if (rc) return rc;
    uint32_t flags = 0;
    CUDA_TRY(launch_kwpir_check(keys, n, d_sorted.ptr, d_temp.ptr, temp_bytes, d_words.ptr, st));
    CUDA_TRY(cudaMemcpyAsync(&flags, d_words.ptr, sizeof flags, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (flags & KWPIR_RESERVED) return fail(B200DPF_EINVAL, "keyword 2^64 - 1 is reserved (tag 0 marks an empty slot)");
    if (flags & KWPIR_DUPLICATE) return fail(B200DPF_EINVAL, "duplicate keywords: each keyword may appear once");
    d_sorted.release();
    d_temp.release();

    DeviceBuffer<unsigned long long> d_bid;
    DeviceBuffer<int32_t> d_owner;
    DeviceBuffer<uint8_t> d_choice;
    DeviceBuffer<uint32_t> d_list[2];
    rc = d_bid.reserve(slots * sizeof(unsigned long long));
    if (!rc) rc = d_owner.reserve(slots * sizeof(int32_t));
    if (!rc) rc = d_choice.reserve(n);
    if (!rc) rc = d_list[0].reserve(n * sizeof(uint32_t));
    if (!rc) rc = d_list[1].reserve(n * sizeof(uint32_t));
    if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(d_bid.ptr, 0, slots * sizeof(unsigned long long), st));   /* round 0: below every bid */
    CUDA_TRY(cudaMemsetAsync(d_owner.ptr, 0xff, slots * sizeof(int32_t), st));          /* -1: empty */
    CUDA_TRY(cudaMemsetAsync(d_choice.ptr, 0, n, st));
    cudaEvent_t ev[2] = {nullptr, nullptr};
    CUDA_TRY(cudaEventCreate(&ev[0]));
    cudaError_t e = cudaEventCreate(&ev[1]);
    uint32_t homeless = (uint32_t)n;
    int round = 0;
    if (e == cudaSuccess) e = cudaEventRecord(ev[0], st);
    while (e == cudaSuccess && homeless > 0 && round < KWPIR_MAX_ROUNDS) {
        round++;   /* round 1's homeless are all items, in order (a null list) */
        const uint32_t *cur = round == 1 ? nullptr : d_list[round & 1].ptr;
        uint32_t *next = d_list[(round + 1) & 1].ptr;
        e = cudaMemsetAsync(d_words.ptr + 1, 0, sizeof(uint32_t), st);
        if (e == cudaSuccess)
            e = launch_kwpir_round(L, keys, cur, homeless, (uint32_t)round, d_choice.ptr, d_bid.ptr, d_owner.ptr, next, d_words.ptr + 1, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(&homeless, d_words.ptr + 1, sizeof homeless, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (e == cudaSuccess) e = cudaEventRecord(ev[1], st);
    if (e == cudaSuccess) e = cudaEventSynchronize(ev[1]);
    float ms = 0.f;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, ev[0], ev[1]);
    cudaEventDestroy(ev[0]);
    if (ev[1]) cudaEventDestroy(ev[1]);
    CUDA_TRY(e);
    if (homeless > 0)
        return fail(B200DPF_EFULL, "placement left %u of %llu items homeless after %d rounds (m=%llu, layout_seed=%llu): use another "
                    "seed or a larger m", homeless, (unsigned long long)n, round, (unsigned long long)L.m, (unsigned long long)L.seed);
    d_bid.release();
    d_owner.release();
    d_list[0].release();
    d_list[1].release();

    /* write_rows waits: the scratch is free after it */
    rc = write_rows(c, values, n, L.value_size, RowPlacement{}, [&](const int32_t *chunk, uint64_t first, uint64_t count) {
        return launch_kwpir_scatter(chunk, first, count, keys, d_choice.ptr, L, c->bins->d_place.ptr, c->d_table.ptr, c->entry_pad, st);
    });
    if (rc) return rc;
    *K = GroupBins::Keyword{L, round, ms};
    return B200DPF_OK;
}

int b200dpf_kwpir_create(b200dpf_ctx **out, const uint64_t *keywords, const int32_t *values, int64_t n, int value_size, int64_t m,
                         uint64_t layout_seed, int device, int kind)
{
    if (!out) return fail(B200DPF_EINVAL, "null ctx out pointer");
    *out = nullptr;
    if (!keywords || !values) return fail(B200DPF_EINVAL, "null buffer");
    KeywordLayout L;
    int rc = kwpir_layout_of(n, value_size, m, layout_seed, &L);
    if (rc) return rc;
    const int64_t rows[KWPIR_TABLES] = {m, m, m};
    std::optional<DeviceGuard> guard;
    std::unique_ptr<b200dpf_ctx> c;
    rc = group_open(nullptr, rows, KWPIR_TABLES, value_size + 2, device, kind, true, &guard, &c);
    if (rc) return rc;
    GroupBins::Keyword K;
    rc = kwpir_build(c.get(), keywords, values, L, &K);
    if (rc) return rc;
    c->bins->keyword = K;
    *out = c.release();
    return B200DPF_OK;
}

int b200dpf_kwpir_layout(const b200dpf_ctx *c, int64_t *n, int64_t *m, uint64_t *seed, int *value_size)
{
    const GroupBins::Keyword *K = nullptr;
    const int rc = kwpir_of(c, &K);
    if (rc) return rc;
    if (!n || !m || !seed || !value_size) return fail(B200DPF_EINVAL, "null buffer");
    *n = (int64_t)K->layout.n;
    *m = (int64_t)K->layout.m;
    *seed = K->layout.seed;
    *value_size = K->layout.value_size;
    return B200DPF_OK;
}

int b200dpf_kwpir_build_stats(const b200dpf_ctx *c, int *rounds, double *place_ms)
{
    const GroupBins::Keyword *K = nullptr;
    const int rc = kwpir_of(c, &K);
    if (rc) return rc;
    if (!rounds || !place_ms) return fail(B200DPF_EINVAL, "null buffer");
    *rounds = K->rounds;
    *place_ms = K->place_ms;
    return B200DPF_OK;
}

int b200dpf_kwpir_locate(int64_t m, uint64_t layout_seed, const uint64_t *keywords, int64_t count, int64_t *rows3)
{
    int rc = kwpir_check_m(m);
    if (rc) return rc;
    if (count < 0) return fail(B200DPF_EINVAL, "count=%lld is negative", (long long)count);
    if (count > 0 && (!keywords || !rows3)) return fail(B200DPF_EINVAL, "null buffer");
    rc = kwpir_reserved(keywords, count);
    if (rc) return rc;
    const KeywordLayout L{0, (uint64_t)m, layout_seed, 0};
    for (int64_t j = 0; j < count; j++)
        for (int t = 0; t < KWPIR_TABLES; t++) rows3[j * KWPIR_TABLES + t] = (int64_t)L.row(t, keywords[j]);
    return B200DPF_OK;
}

/* The locator of b200dpf_kwpir_locate, one thread per query, in the caller's buffers only: like
 * b200dpf_batchcode_plan_device it neither joins the context's one-operation-in-flight chain nor reads the context on
 * the device. */
int b200dpf_kwpir_plan_device(b200dpf_ctx *c, const uint64_t *keywords_dev, int64_t nqueries, int64_t *alphas_dev, void *cuda_stream)
{
    const GroupBins::Keyword *K = nullptr;
    int rc = kwpir_of(c, &K);
    if (rc) return rc;
    if (!keywords_dev || !alphas_dev) return fail(B200DPF_EINVAL, "null buffer");
    if (nqueries < 1 || nqueries > ((int64_t)1 << 24) / KWPIR_TABLES)
        return fail(B200DPF_EINVAL, "nqueries=%lld out of range: 1 <= nqueries * 3 <= 2^24", (long long)nqueries);
    if (((reinterpret_cast<uintptr_t>(keywords_dev) | reinterpret_cast<uintptr_t>(alphas_dev)) & 7u) != 0)
        return fail(B200DPF_EINVAL, "keywords_dev and alphas_dev must be 8-byte aligned");
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    CUDA_TRY(launch_kwpir_plan(K->layout, keywords_dev, nqueries, alphas_dev, reinterpret_cast<cudaStream_t>(cuda_stream)));
    return B200DPF_OK;
}

/* The slot of every keyword, found on the device from the tags of its three candidate rows, then the new rows
 * (value and the unchanged tag) through the grouped update path. */
int b200dpf_kwpir_update(b200dpf_ctx *c, const uint64_t *keywords, const int32_t *values, int64_t count)
{
    const GroupBins::Keyword *K = nullptr;
    int rc = kwpir_of(c, &K);
    if (!rc) rc = check_update_args(c, keywords, values, count);
    if (!rc) rc = kwpir_reserved(keywords, count);
    if (rc) return rc;
    if (count == 0) return B200DPF_OK;
    const KeywordLayout &L = K->layout;
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    DeviceBuffer<uint64_t> d_kw;
    DeviceBuffer<int64_t> d_rows;
    DeviceBuffer<int32_t> d_bins;
    rc = d_kw.reserve((size_t)count * sizeof(uint64_t));
    if (!rc) rc = d_rows.reserve((size_t)count * sizeof(int64_t));
    if (!rc) rc = d_bins.reserve((size_t)count * sizeof(int32_t));
    if (rc) return rc;
    std::vector<int32_t> bins((size_t)count);
    std::vector<int64_t> idx((size_t)count);
    /* the tags never change after create, so this lookup needs no ordering against evaluations or updates */
    CUDA_TRY(cudaMemcpyAsync(d_kw.ptr, keywords, (size_t)count * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(launch_kwpir_find(L, d_kw.ptr, count, c->bins->d_place.ptr, c->d_table.ptr, c->entry_pad, d_bins.ptr, d_rows.ptr, c->stream));
    CUDA_TRY(cudaMemcpyAsync(bins.data(), d_bins.ptr, (size_t)count * sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaMemcpyAsync(idx.data(), d_rows.ptr, (size_t)count * sizeof(int64_t), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (int64_t j = 0; j < count; j++)
        if (bins[(size_t)j] < 0)
            return fail(B200DPF_EINVAL, "update %lld: keyword %llu is not in the table", (long long)j, (unsigned long long)keywords[j]);
    const size_t E = (size_t)L.value_size, W = E + 2;
    std::vector<int32_t> rows((size_t)count * W);
    for (int64_t j = 0; j < count; j++) {
        int32_t *r = rows.data() + (size_t)j * W;
        std::memcpy(r, values + (size_t)j * E, E * sizeof(int32_t));
        const uint64_t tag = keywords[j] + 1;
        r[E] = (int32_t)(uint32_t)tag;
        r[E + 1] = (int32_t)(uint32_t)(tag >> 32);
    }
    rc = update_host_enqueue(c, idx.data(), bins.data(), rows.data(), count);
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    return B200DPF_OK;
}

int b200dpf_kwpir_tags(const b200dpf_ctx *c, uint64_t *tags)
{
    const GroupBins::Keyword *K = nullptr;
    const int rc = kwpir_of(c, &K);
    if (rc) return rc;
    if (!tags) return fail(B200DPF_EINVAL, "null buffer");
    const uint64_t m = K->layout.m;
    DeviceGuard guard(c->device);
    if (!guard.ok) return fail(B200DPF_ECUDA, "cudaSetDevice(%d) failed", c->device);
    const size_t pitch = (size_t)c->entry_pad * sizeof(int32_t);
    for (int t = 0; t < KWPIR_TABLES; t++) {
        const int32_t *src = c->d_table.ptr + c->bins->shape[(size_t)t].first * (uint64_t)c->entry_pad + K->layout.value_size;
        CUDA_TRY(cudaMemcpy2DAsync(tags + (size_t)t * m, sizeof(uint64_t), src, pitch, sizeof(uint64_t), (size_t)m,
                                   cudaMemcpyDeviceToHost, c->stream));
    }
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

int b200dpf_group_bins(const b200dpf_ctx *c) { return (c && c->bins) ? (int)c->bins->shape.size() : 0; }

int64_t b200dpf_ctx_table_rows(const b200dpf_ctx *c)
{
    if (!c) return -1;
    return (c->multi ? c->multi->sub[0] : c)->rows_local();
}


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
