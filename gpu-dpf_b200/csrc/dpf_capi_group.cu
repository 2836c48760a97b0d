/* ------------------------------------------------------------------------------------------- */
/* Grouped evaluation: the batch-PIR front end (SURVEY.md section 8(f) rank 4).                  */
/* ------------------------------------------------------------------------------------------- */

#include "dpf_ctx.h"

#include <new>

namespace b200dpf::capi {

/* The context every grouped create function starts from: bins of n[g] rows for keys of `kind`, their shapes,
 * placements and per-bin tables on the device (enqueued on the context's stream), and a zeroed device table, current
 * while `guard` lives.  `tables` (null: not checked) are the bins' sources.  n and the row offsets count rows, the
 * depths (per bin and the context's deepest) leaves. */
int group_open(const int32_t *const *tables, const int64_t *n, int nbins, int entry_size, int device, int kind,
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

}  // namespace b200dpf::capi

extern "C" {

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

}  // extern "C"
