/*
 * dpf_capi.cu -- implementation of the C ABI declared in include/b200dpf.h.
 *
 * Owns the device state of one table (or one entry-range shard of it) and
 * turns b200dpf_eval* calls into launches of the sm_90a kernel in
 * dpf_kernels.cu.  The GPU entry points have no CPU fallback: without a usable
 * CUDA device they fail with B200DPF_ECUDA.
 *
 * The other entry-point families live in dpf_capi_keys.cu, dpf_capi_multi.cu, dpf_capi_group.cu,
 * dpf_capi_update.cu, dpf_capi_batchcode.cu and dpf_capi_kwpir.cu, the planner and launcher in dpf_plan.cu,
 * and what they share (the context among it) in dpf_ctx.h.
 */
#include "dpf_ctx.h"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <new>

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

int env_int(const char *name, int dflt)
{
    const char *v = std::getenv(name);
    return (v && *v) ? std::atoi(v) : dflt;
}

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

/* "a standard", "an early-terminated", "an XOR-shared": the article of a kind's name */
inline const char *article(int kind) { return kind == host::KIND_STANDARD ? "a" : "an"; }

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

}  // namespace

b200dpf_ctx::Knobs::Knobs() { for (const KnobInfo &k : kKnobs) this->*k.field = k.dflt; }

b200dpf_ctx::~b200dpf_ctx()
{
    if (ev_done) cudaEventDestroy(ev_done);
    if (ev_t0) cudaEventDestroy(ev_t0);
    if (ev_t1) cudaEventDestroy(ev_t1);
    if (stream) cudaStreamDestroy(stream);
}

namespace b200dpf::capi {

thread_local char g_err[512] = "";

int fail(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
    return code;
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

/* Write the rows of placement P from `src`, the caller's table of P.n rows, padded to 64-byte rows */
int fill_table(b200dpf_ctx *c, const int32_t *src, const RowPlacement &P, DeviceBuffer<int32_t> *keep)
{
    return write_rows(c, src, P.n, c->entry_size, P, [&](const int32_t *chunk, uint64_t first, uint64_t count) {
        return launch_fill_table(chunk, first, count, c->d_table.ptr, P, c->entry_size, c->entry_pad, c->sm_count, c->stream);
    }, keep);
}

}  // namespace b200dpf::capi

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

const char *b200dpf_version(void) { return "b200dpf 0.1.0 sm_90a"; }

const char *b200dpf_last_error(void) { return g_err; }

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
