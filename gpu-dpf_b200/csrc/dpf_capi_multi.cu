/* ------------------------------------------------------------------------------------------- */
/* One process, several GPUs (SURVEY.md section 2.2 / 8(b): "single process drives 1/2/4/8 GPUs"). */
/* ------------------------------------------------------------------------------------------- */
/* MultiState (dpf_ctx.h) holds the sub-contexts and worker threads of one such context. */

#include "dpf_ctx.h"

#include <new>

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

namespace b200dpf::capi {

b200dpf_ctx *multi_first(b200dpf_ctx *root) { return root->multi->sub[0]; }

int multi_last_launches(const b200dpf_ctx *root)
{
    int total = 0;
    for (const b200dpf_ctx *c : root->multi->sub) total += c->last_launches;
    return total;
}

int multi_set_option(b200dpf_ctx *root, const char *name, int value)
{
    for (b200dpf_ctx *c : root->multi->sub) {
        const int rc = b200dpf_ctx_set_option(c, name, value);
        if (rc) return rc;
    }
    return B200DPF_OK;
}

int multi_eval_host(b200dpf_ctx *root, const void *keys, size_t key_stride_bytes, const KeyLayout &kl, int64_t nkeys,
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

}  // namespace b200dpf::capi

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

}  // extern "C"
