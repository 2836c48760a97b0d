/* ------------------------------------------------------------------------------------------- */
/* Keyword PIR: a value by its 64-bit keyword in one query (DESIGN.md section 14).               */
/* ------------------------------------------------------------------------------------------- */

#include "dpf_ctx.h"

extern "C" {

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

}  // extern "C"
