/*
 * dpf_kwpir.cu -- the kernels of keyword-PIR contexts (b200dpf_kwpir_create, DESIGN.md section 14): the duplicate
 * check, the rounds of the deterministic cuckoo placement, the scatter that writes each item's row into its slot, the
 * client's locator for load generators (b200dpf_kwpir_plan_device) and the slot lookup of row updates.  All of them
 * place keywords through KeywordLayout (dpf_kernels.cuh); the evaluation kernels are not involved.
 */
#include <cub/cub.cuh>

#include "dpf_kernels.cuh"

namespace b200dpf {

namespace {

constexpr int kThreads = 256;        /* threads per block: one item, query or keyword each */
constexpr int kScatterWarps = 8;     /* warps per block: one item each */

unsigned blocks_for(uint64_t count, int per_block) { return (unsigned)((count + per_block - 1) / per_block); }

__global__ void __launch_bounds__(kThreads) kwpir_check_kernel(const uint64_t *__restrict__ sorted, uint64_t n,
                                                               uint32_t *__restrict__ flags)
{
    const uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    if (i + 1 < n && sorted[i] == sorted[i + 1]) atomicOr(flags, (uint32_t)KWPIR_DUPLICATE);
    if (sorted[i] == ~0ull) atomicOr(flags, (uint32_t)KWPIR_RESERVED);
}

/* The slot item i bids for this round: its current table's candidate */
__device__ __forceinline__ uint64_t bid_slot(const KeywordLayout &L, const uint64_t *keys, const uint8_t *choice, uint32_t i)
{
    const int c = choice[i];
    return (uint64_t)c * L.m + L.row(c, keys[i]);
}

__global__ void __launch_bounds__(kThreads) kwpir_bid_kernel(const KeywordLayout L, const uint64_t *__restrict__ keys,
                                                             const uint32_t *__restrict__ homeless, uint32_t count,
                                                             uint32_t round, const uint8_t *__restrict__ choice,
                                                             unsigned long long *__restrict__ bid)
{
    const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
    if (t >= count) return;
    const uint32_t i = homeless ? homeless[t] : t;
    atomicMax(&bid[bid_slot(L, keys, choice, i)], (unsigned long long)round << 32 | (uint32_t)~i);
}

/* Every bid of this round is in: the winner of each slot takes it (one winner per slot, so owner[s] has one writer),
 * and the loser -- a bidder that did not win, or the owner a winner evicted -- moves on to its next table.  Neither
 * is touched by any other thread this round: an evicted owner was not homeless, so it did not bid. */
__global__ void __launch_bounds__(kThreads) kwpir_resolve_kernel(const KeywordLayout L, const uint64_t *__restrict__ keys,
                                                                 const uint32_t *__restrict__ homeless, uint32_t count,
                                                                 uint32_t round, uint8_t *__restrict__ choice,
                                                                 const unsigned long long *__restrict__ bid,
                                                                 int32_t *__restrict__ owner, uint32_t *__restrict__ next,
                                                                 uint32_t *__restrict__ next_count)
{
    const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
    if (t >= count) return;
    const uint32_t i = homeless ? homeless[t] : t;
    const uint64_t s = bid_slot(L, keys, choice, i);
    uint32_t loser = i;
    if (bid[s] == ((unsigned long long)round << 32 | (uint32_t)~i)) {
        const int32_t old = owner[s];
        owner[s] = (int32_t)i;
        if (old < 0) return;
        loser = (uint32_t)old;
    }
    choice[loser] = (uint8_t)((choice[loser] + 1) % KWPIR_TABLES);
    next[atomicAdd(next_count, 1u)] = loser;
}

__global__ void __launch_bounds__(kScatterWarps * 32) kwpir_scatter_kernel(const int32_t *__restrict__ values, uint64_t first,
                                                                           uint64_t count, const uint64_t *__restrict__ keys,
                                                                           const uint8_t *__restrict__ choice, const KeywordLayout L,
                                                                           const RowPlacement *__restrict__ place,
                                                                           int32_t *__restrict__ table, int stride)
{
    const uint64_t w = (uint64_t)blockIdx.x * kScatterWarps + (threadIdx.x >> 5);
    if (w >= count) return;
    const int lane = threadIdx.x & 31;
    const uint64_t key = keys[first + w];
    const int c = choice[first + w];
    int32_t *t = table + (place[c].first + L.row(c, key)) * (uint64_t)stride;
    const int32_t *s = values + w * (uint64_t)L.value_size;
    for (int col = lane; col < L.value_size; col += 32) t[col] = s[col];
    if (lane == 0) {
        const uint64_t tag = key + 1;
        t[L.value_size] = (int32_t)(uint32_t)tag;
        t[L.value_size + 1] = (int32_t)(uint32_t)(tag >> 32);
    }
}

__global__ void __launch_bounds__(kThreads) kwpir_plan_kernel(const KeywordLayout L, const uint64_t *__restrict__ keywords,
                                                              int64_t nq, int64_t *__restrict__ rows3)
{
    const int64_t q = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (q >= nq) return;
    const uint64_t w = keywords[q];
    for (int c = 0; c < KWPIR_TABLES; c++) rows3[q * KWPIR_TABLES + c] = (int64_t)L.row(c, w);
}

__global__ void __launch_bounds__(kThreads) kwpir_find_kernel(const KeywordLayout L, const uint64_t *__restrict__ keywords,
                                                              int64_t count, const RowPlacement *__restrict__ place,
                                                              const int32_t *__restrict__ table, int stride,
                                                              int32_t *__restrict__ bins, int64_t *__restrict__ rows)
{
    const int64_t j = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (j >= count) return;
    const uint64_t w = keywords[j];
    int32_t bin = -1;
    int64_t row = -1;
    for (int c = 0; c < KWPIR_TABLES; c++) {
        const uint64_t r = L.row(c, w);
        const int32_t *t = table + (place[c].first + r) * (uint64_t)stride + L.value_size;
        const uint64_t tag = (uint64_t)(uint32_t)t[0] | (uint64_t)(uint32_t)t[1] << 32;
        if (tag == w + 1) {
            bin = c;
            row = (int64_t)r;
        }
    }
    bins[j] = bin;
    rows[j] = row;
}

}  // namespace

cudaError_t kwpir_check_temp_bytes(uint64_t n, size_t *bytes)
{
    *bytes = 0;
    return cub::DeviceRadixSort::SortKeys(nullptr, *bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr, (int)n);
}

cudaError_t launch_kwpir_check(const uint64_t *keys, uint64_t n, uint64_t *sorted, void *temp, size_t temp_bytes, uint32_t *flags,
                               cudaStream_t stream)
{
    cudaError_t e = cudaMemsetAsync(flags, 0, sizeof(uint32_t), stream);
    if (e == cudaSuccess) e = cub::DeviceRadixSort::SortKeys(temp, temp_bytes, keys, sorted, (int)n, 0, 64, stream);
    if (e != cudaSuccess) return e;
    kwpir_check_kernel<<<blocks_for(n, kThreads), kThreads, 0, stream>>>(sorted, n, flags);
    return cudaGetLastError();
}

cudaError_t launch_kwpir_round(const KeywordLayout &L, const uint64_t *keys, const uint32_t *homeless, uint32_t count,
                               uint32_t round, uint8_t *choice, unsigned long long *bid, int32_t *owner, uint32_t *next,
                               uint32_t *next_count, cudaStream_t stream)
{
    const unsigned grid = blocks_for(count, kThreads);
    kwpir_bid_kernel<<<grid, kThreads, 0, stream>>>(L, keys, homeless, count, round, choice, bid);
    kwpir_resolve_kernel<<<grid, kThreads, 0, stream>>>(L, keys, homeless, count, round, choice, bid, owner, next, next_count);
    return cudaGetLastError();
}

cudaError_t launch_kwpir_scatter(const int32_t *values, uint64_t first, uint64_t count, const uint64_t *keys, const uint8_t *choice,
                                 const KeywordLayout &L, const RowPlacement *place, int32_t *table, int stride, cudaStream_t stream)
{
    if (count == 0) return cudaSuccess;
    kwpir_scatter_kernel<<<blocks_for(count, kScatterWarps), kScatterWarps * 32, 0, stream>>>(values, first, count, keys, choice, L,
                                                                                               place, table, stride);
    return cudaGetLastError();
}

cudaError_t launch_kwpir_plan(const KeywordLayout &L, const uint64_t *keywords, int64_t nq, int64_t *rows3, cudaStream_t stream)
{
    kwpir_plan_kernel<<<blocks_for((uint64_t)nq, kThreads), kThreads, 0, stream>>>(L, keywords, nq, rows3);
    return cudaGetLastError();
}

cudaError_t launch_kwpir_find(const KeywordLayout &L, const uint64_t *keywords, int64_t count, const RowPlacement *place,
                              const int32_t *table, int stride, int32_t *bins, int64_t *rows, cudaStream_t stream)
{
    kwpir_find_kernel<<<blocks_for((uint64_t)count, kThreads), kThreads, 0, stream>>>(L, keywords, count, place, table, stride,
                                                                                      bins, rows);
    return cudaGetLastError();
}

}  // namespace b200dpf
