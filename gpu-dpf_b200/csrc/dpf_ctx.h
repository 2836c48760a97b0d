/*
 * dpf_ctx.h -- private to the implementation of the C ABI (dpf_capi*.cu, dpf_plan.cu); not installed.
 *
 * The context, the launch-plan types and the helpers that more than one of those files calls.  A helper
 * that one file alone uses stays in that file.
 */
#pragma once

#include "b200dpf.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstring>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "dpf_host.h"
#include "dpf_kernels.cuh"

namespace b200dpf::capi {

/* the calling thread's last error text (b200dpf_last_error): defined once, in dpf_capi.cu */
extern thread_local char g_err[512];

int fail(int code, const char *fmt, ...);

#define CUDA_TRY(expr)                                                                        \
    do {                                                                                      \
        cudaError_t e__ = (expr);                                                             \
        if (e__ != cudaSuccess)                                                               \
            return fail(B200DPF_ECUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e__),       \
                        __FILE__, __LINE__);                                                  \
    } while (0)

inline int ilog2(int64_t v)
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

struct SmemLayout {
    int threads, blocks_per_sm, grid;
    int budget;               /* dynamic shared memory one block may use */
    size_t smem_fixed;        /* AES: whole budget; others: computed from s */
    uint32_t off_meta;        /* correction words, meta_cw bytes                          */
    uint32_t off_small;       /* level-0 low words, root seeds and flag (kMetaSmall bytes) */
    uint32_t off_lo, off_hi, off_tab, meta_cw, level_bytes;
    int cap_lo, cap_hi, s_max;
};

/* per (prf, nv, mode) launch layouts, filled on first use */
struct SmemLayoutCache {
    SmemLayout entry[4][3][MODE_COUNT];
    bool valid[4][3][MODE_COUNT] = {};
};

struct MultiState;        /* b200dpf_create_multi: per-device sub-contexts + worker threads */
struct GroupBins;         /* b200dpf_group_create: many tables ("bins") behind one context */

}  // namespace b200dpf::capi

/* every file of the C ABI's implementation works in both namespaces */
using namespace b200dpf;
using namespace b200dpf::capi;

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

namespace b200dpf::capi {

/* Where the kernel finds the live parts of a key. */
struct KeyLayout {
    uint32_t stride_v, root_v;
    int compact;
};
inline KeyLayout reference_layout() { return KeyLayout{131u, 129u, 0}; }                       /* dpf_wrapper.cu:26-46 */
inline KeyLayout compact_layout(int depth) { return KeyLayout{2u + 4u * (uint32_t)depth, 1u, 1}; }   /* b200dpf_key_pack */

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

/* The work-item size of a key group of bin g on a grouped context */
inline int group_s(const EvalPlan &P, const GroupBins &B, int g) { return std::max(1, std::min(B.shape[(size_t)g].room, P.s_group)); }

constexpr int64_t kMaxUpdateCount = 0x7fffffff;   /* occurrence numbers are 32-bit, as is the sort's item count */

/* ---- dpf_capi.cu: the context's set-up, its one-operation-in-flight chain, staging and key checks ---- */

int wait_last(b200dpf_ctx *c, cudaStream_t stream);
int mark_last(b200dpf_ctx *c, cudaStream_t stream);
int reserve_host_keys(b200dpf_ctx *c, size_t key_bytes);
int reserve_host_out(b200dpf_ctx *c, size_t out_elems);
int reserve_device_io(b200dpf_ctx *c, size_t key_bytes, size_t out_elems);
int table_shape(int64_t n, int kind, bool trimmed, int bin, TableShape *t);
RowPlacement place_of(const TableShape &t, int lane_bits, bool trimmed, int rank, int shard_bits);
int check_key(const b200dpf_ctx *c, const TableShape &t, const int32_t *key, int64_t b, int bin);
bool is_pinned_host(const void *ptr);
int download_out(b200dpf_ctx *c, int32_t *out, bool out_pinned, size_t elems);
int open_device(int device, const char *cpu_hint, std::optional<DeviceGuard> *guard);
int ctx_open(int device, bool read_env, std::optional<DeviceGuard> *guard, std::unique_ptr<b200dpf_ctx> *out);
int wait_source(const b200dpf_ctx *c, const void *src, bool *on_device, int *src_device);
int fill_table(b200dpf_ctx *c, const int32_t *src, const RowPlacement &P, DeviceBuffer<int32_t> *keep = nullptr);

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

/* ---- dpf_plan.cu: shared-memory layouts, the planners and the launcher ---- */

int smem_layout(b200dpf_ctx *c, int prf, int nv, int mode, SmemLayout *L);
int plan_group_eval(b200dpf_ctx *c, int prf, const std::vector<int64_t> &count, EvalPlan *out);
int plan_group_device(b200dpf_ctx *c, int prf, int64_t nkeys, DevicePlanned *D);
int launch_plan(b200dpf_ctx *c, const EvalJob &J, const EvalPlan &P);
int run_pipeline(b200dpf_ctx *c, const void *keys_dev, const KeyLayout &kl, int64_t nkeys, int prf, int mode_main,
                 void *out_dev, cudaStream_t stream, bool clear_out = true);

/* ---- dpf_capi_multi.cu: multi-device contexts ---- */

b200dpf_ctx *multi_first(b200dpf_ctx *root);
int multi_last_launches(const b200dpf_ctx *root);
int multi_set_option(b200dpf_ctx *root, const char *name, int value);
int multi_eval_host(b200dpf_ctx *root, const void *keys, size_t key_stride_bytes, const KeyLayout &kl, int64_t nkeys,
                    int prf, int32_t *out);

/* ---- dpf_capi_group.cu: grouped contexts ---- */

int group_open(const int32_t *const *tables, const int64_t *n, int nbins, int entry_size, int device, int kind,
               bool trimmed, std::optional<DeviceGuard> *guard, std::unique_ptr<b200dpf_ctx> *out);

/* ---- dpf_capi_update.cu: row updates ---- */

int update_host_enqueue(b200dpf_ctx *c, const int64_t *idx, const int32_t *bins, const int32_t *rows, int64_t count);
int check_update_args(const b200dpf_ctx *c, const void *idx, const void *rows, int64_t count);

}  // namespace b200dpf::capi
