/*
 * dpf_group_io.cu -- the per-key work of a device-resident grouped evaluation (b200dpf_group_eval_device
 * and b200dpf_group_eval_queries_device): the gathers that put the caller's keys (wire format, or queries of
 * compact keys) into bin order, in the compact layout the grouped kernels read, and the scatter that puts the
 * bin-ordered results back into the caller's order.  They replace host loops of b200dpf_group_eval
 * (pack_compact and the final reorder); the evaluation kernels are not involved.
 */
#include "dpf_host.h"
#include "dpf_kernels.cuh"

namespace b200dpf {

namespace {

constexpr int kIoWarps = 8;                                     /* warps per block: one key each */
constexpr uint32_t kWireSlots = host::KEY_WORDS / 4;            /* 131 uint4 per wire-format key */

/* compact[pos] = pack_compact(keys[order[pos].x], depth order[pos].y): slot 0 = (magic, depth, 0, 0), slot 1
 * = the root, then per level L the four slots cw_1[L] (two) and cw_2[L] (two).  Slots past the key's own
 * levels are not written, as on the host. */
__global__ void __launch_bounds__(kIoWarps * 32) group_gather_kernel(const uint4 *__restrict__ keys,
                                                                     const uint2 *__restrict__ order, int64_t nkeys,
                                                                     uint32_t magic, uint32_t stride_v,
                                                                     uint4 *__restrict__ compact)
{
    const int64_t pos = (int64_t)blockIdx.x * kIoWarps + (threadIdx.x >> 5);
    if (pos >= nkeys) return;
    const uint2 o = order[pos];
    const uint4 *k = keys + (size_t)o.x * kWireSlots;
    uint4 *d = compact + (size_t)pos * stride_v;
    const uint32_t slots = 2u + 4u * o.y;
    for (uint32_t j = threadIdx.x & 31; j < slots; j += 32) {
        uint4 v;
        if (j == 0) {
            v = make_uint4(magic, o.y, 0u, 0u);
        } else if (j == 1) {
            v = k[host::SLOT_ROOT];
        } else {
            const uint32_t level = (j - 2) >> 2, w = (j - 2) & 3;
            v = k[(w < 2 ? host::SLOT_CW1 : host::SLOT_CW2) + 2 * level + (w & 1)];
        }
        d[j] = v;
    }
}

/* out[order[pos].x][c] = sorted[pos][c] for c < entry_size */
__global__ void __launch_bounds__(kIoWarps * 32) group_scatter_kernel(const uint32_t *__restrict__ sorted,
                                                                      const uint2 *__restrict__ order, int64_t nkeys,
                                                                      int entry_size, uint32_t *__restrict__ out)
{
    const int64_t pos = (int64_t)blockIdx.x * kIoWarps + (threadIdx.x >> 5);
    if (pos >= nkeys) return;
    const uint32_t *s = sorted + (size_t)pos * entry_size;
    uint32_t *d = out + (size_t)order[pos].x * entry_size;
    for (int c = threadIdx.x & 31; c < entry_size; c += 32) d[c] = s[c];
}

/* compact[pos] = key g of query q for pos = g * nq + q: the compact key at uint4 offset q * query_v + bins[g].x
 * of `queries`, which is already in the layout pack_compact writes, with slot 0 rewritten to (magic, depth, 0,
 * 0) -- its own header is not read.  Slots past the key's own levels are neither read nor written. */
__global__ void __launch_bounds__(kIoWarps * 32) group_gather_queries_kernel(const uint4 *__restrict__ queries,
                                                                             const uint2 *__restrict__ bins, int64_t nkeys,
                                                                             uint32_t nq, uint64_t query_v, uint32_t magic,
                                                                             uint32_t stride_v, uint4 *__restrict__ compact)
{
    const int64_t pos = (int64_t)blockIdx.x * kIoWarps + (threadIdx.x >> 5);
    if (pos >= nkeys) return;
    const uint32_t g = (uint32_t)pos / nq, q = (uint32_t)pos - g * nq;
    const uint2 b = bins[g];
    const uint4 *k = queries + (size_t)q * query_v + b.x;
    uint4 *d = compact + (size_t)pos * stride_v;
    const uint32_t slots = 2u + 4u * b.y;
    for (uint32_t j = threadIdx.x & 31; j < slots; j += 32) d[j] = j == 0 ? make_uint4(magic, b.y, 0u, 0u) : k[j];
}

}  // namespace

cudaError_t launch_group_gather_queries(const void *queries, const uint2 *bins, int64_t nkeys, uint32_t nq, uint64_t query_v,
                                        uint32_t magic, uint32_t stride_v, void *compact, cudaStream_t stream)
{
    const unsigned grid = (unsigned)((nkeys + kIoWarps - 1) / kIoWarps);
    group_gather_queries_kernel<<<grid, kIoWarps * 32, 0, stream>>>(reinterpret_cast<const uint4 *>(queries), bins, nkeys, nq,
                                                                    query_v, magic, stride_v, reinterpret_cast<uint4 *>(compact));
    return cudaGetLastError();
}

cudaError_t launch_group_gather(const void *keys, const uint2 *order, int64_t nkeys, uint32_t magic, uint32_t stride_v,
                                void *compact, cudaStream_t stream)
{
    const unsigned grid = (unsigned)((nkeys + kIoWarps - 1) / kIoWarps);
    group_gather_kernel<<<grid, kIoWarps * 32, 0, stream>>>(reinterpret_cast<const uint4 *>(keys), order, nkeys, magic,
                                                            stride_v, reinterpret_cast<uint4 *>(compact));
    return cudaGetLastError();
}

cudaError_t launch_group_scatter(const int32_t *sorted, const uint2 *order, int64_t nkeys, int entry_size, void *out,
                                 cudaStream_t stream)
{
    const unsigned grid = (unsigned)((nkeys + kIoWarps - 1) / kIoWarps);
    group_scatter_kernel<<<grid, kIoWarps * 32, 0, stream>>>(reinterpret_cast<const uint32_t *>(sorted), order, nkeys,
                                                             entry_size, reinterpret_cast<uint32_t *>(out));
    return cudaGetLastError();
}

}  // namespace b200dpf
