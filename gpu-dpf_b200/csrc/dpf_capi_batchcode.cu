/* ------------------------------------------------------------------------------------------- */
/* Batch codes: any k rows of one table per query (DESIGN.md section 13).                        */
/* ------------------------------------------------------------------------------------------- */

#include "dpf_ctx.h"

extern "C" {

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

}  // extern "C"
