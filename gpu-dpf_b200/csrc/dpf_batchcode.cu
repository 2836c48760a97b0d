/*
 * dpf_batchcode.cu -- the kernels of batch-code contexts (b200dpf_batchcode_create, DESIGN.md section 13): the scatter
 * that writes each table row's three copies into their bins at create, and the client's planner for load generators
 * (b200dpf_batchcode_plan_device).  Both place rows through BatchCodeLayout (dpf_kernels.cuh); the evaluation kernels
 * are not involved.
 */
#include "dpf_kernels.cuh"

namespace b200dpf {

namespace {

constexpr int kScatterWarps = 8;     /* warps per block: one table row each */
constexpr int kPlanThreads = 128;    /* threads per block: one query each */

/* Row first + w of the table, at src[w]: lanes 0..2 find copies 0..2, then the warp writes the row to all three, the
 * columns of a row side by side. */
__global__ void __launch_bounds__(kScatterWarps * 32) batchcode_scatter_kernel(const int32_t *__restrict__ src, uint64_t first,
                                                                              uint64_t count, const BatchCodeLayout L,
                                                                              const RowPlacement *__restrict__ place,
                                                                              int32_t *__restrict__ table, int cols, int stride)
{
    const uint64_t w = (uint64_t)blockIdx.x * kScatterWarps + (threadIdx.x >> 5);
    if (w >= count) return;
    const int lane = threadIdx.x & 31;
    uint64_t dst = 0;
    if (lane < BATCHCODE_COPIES) {
        uint32_t bin;
        uint64_t row;
        L.locate(lane, first + w, &bin, &row);
        dst = place[bin].first + row;
    }
    const uint64_t d0 = __shfl_sync(0xffffffffu, dst, 0), d1 = __shfl_sync(0xffffffffu, dst, 1),
                   d2 = __shfl_sync(0xffffffffu, dst, 2);
    const int32_t *s = src + w * (uint64_t)cols;
    int32_t *t0 = table + d0 * (uint64_t)stride, *t1 = table + d1 * (uint64_t)stride, *t2 = table + d2 * (uint64_t)stride;
    for (int c = lane; c < cols; c += 32) {
        const int32_t v = s[c];
        t0[c] = v;
        t1[c] = v;
        t2[c] = v;
    }
}

__global__ void __launch_bounds__(kPlanThreads) batchcode_plan_kernel(const BatchCodeLayout L, const int64_t *__restrict__ wanted,
                                                                     int64_t nq, int k, int64_t *__restrict__ alphas,
                                                                     int32_t *__restrict__ slots)
{
    const int64_t q = (int64_t)blockIdx.x * kPlanThreads + threadIdx.x;
    if (q >= nq) return;
    batchcode_plan_query(L, wanted + q * k, k, alphas + q * (int64_t)L.nbins, slots + q * k);
}

}  // namespace

cudaError_t launch_batchcode_scatter(const int32_t *src, uint64_t first, uint64_t count, const BatchCodeLayout &L,
                                     const RowPlacement *place, int32_t *table, int cols, int stride, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    const unsigned grid = (unsigned)((count + kScatterWarps - 1) / kScatterWarps);
    batchcode_scatter_kernel<<<grid, kScatterWarps * 32, 0, stream>>>(src, first, count, L, place, table, cols, stride);
    return cudaGetLastError();
}

cudaError_t launch_batchcode_plan(const BatchCodeLayout &L, const int64_t *wanted, int64_t nq, int k, int64_t *alphas,
                                  int32_t *slots, cudaStream_t stream)
{
    const unsigned grid = (unsigned)((nq + kPlanThreads - 1) / kPlanThreads);
    batchcode_plan_kernel<<<grid, kPlanThreads, 0, stream>>>(L, wanted, nq, k, alphas, slots);
    return cudaGetLastError();
}

}  // namespace b200dpf
