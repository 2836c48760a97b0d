/* ------------------------------------------------------------------------------------------- */
/* Row updates of a live table.                                                                  */
/* ------------------------------------------------------------------------------------------- */

#include "dpf_ctx.h"

namespace {

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

}  // namespace

namespace b200dpf::capi {

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

}  // namespace b200dpf::capi

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

}  // extern "C"
