/*
 * dpf_group_plan.cu -- the plan of a grouped evaluation made on the device from a device-resident bin list
 * (b200dpf_group_eval_device_bins).  GroupLaunch::plan makes the same lists on the host from host bins: the sort by
 * bin, the order list, the key groups' descriptors and the work units.  Here the host decides only what needs no key
 * counts (GroupPlanParams); these kernels do the rest on the caller's stream, so the call never waits on the host.
 * The evaluation kernels then read the list lengths from GroupPlanParams::counts (ModeTraits::counts_on_device).
 */
#include <cub/cub.cuh>

#include "dpf_kernels.cuh"

namespace b200dpf {

namespace {

constexpr int kPlanThreads = 1024;      /* the plan kernel is one block */
constexpr int kMaxShrink = 6;           /* shrink_s starts at most at s = 6 (the automatic s) */

/* hist[key]++ for key = bins[b], or nbins when it is out of range; the sort's inputs (key, caller's index).  The
 * lanes of a warp that share a key add once between them: a batch of one bin would otherwise put every key's atomic
 * on one word. */
__global__ void __launch_bounds__(256) group_hist_kernel(const int32_t *__restrict__ bins, int64_t nkeys, int nbins,
                                                         uint32_t *__restrict__ hist, uint32_t *__restrict__ keys_in,
                                                         uint32_t *__restrict__ vals_in)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t b0 = (int64_t)blockIdx.x * blockDim.x; b0 < nkeys; b0 += stride) {
        const int64_t b = b0 + threadIdx.x;
        const bool live = b < nkeys;
        const int32_t g = live ? bins[b] : -1;
        const uint32_t key = (g >= 0 && g < nbins) ? (uint32_t)g : (uint32_t)nbins;
        if (live) {
            keys_in[b] = key;
            vals_in[b] = (uint32_t)b;
        }
        const uint32_t mask = __ballot_sync(0xffffffffu, live);
        if (live) {
            const uint32_t same = __match_any_sync(mask, key);
            if ((threadIdx.x & 31) == (uint32_t)(__ffs(same) - 1)) atomicAdd(hist + key, (uint32_t)__popc(same));
        }
    }
}

/* order[pos] = (caller's index, depth of its bin; 0 for an out-of-range key) */
__global__ void __launch_bounds__(256) group_order_kernel(const uint32_t *__restrict__ keys_out,
                                                          const uint32_t *__restrict__ vals_out, int64_t nkeys, int nbins,
                                                          const GroupBinInfo *__restrict__ info, uint2 *__restrict__ order)
{
    for (int64_t pos = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pos < nkeys; pos += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t g = keys_out[pos];
        order[pos] = make_uint2(vals_out[pos], g < (uint32_t)nbins ? (uint32_t)info[g].depth : 0u);
    }
}

struct PlanSums {
    long long keys, groups, units;
};
struct PlanAdd {
    __device__ PlanSums operator()(const PlanSums &a, const PlanSums &b) const
    {
        return PlanSums{a.keys + b.keys, a.groups + b.groups, a.units + b.units};
    }
};

/* The work-item size of a key group of a bin of `room` (group_s on the host) */
__device__ __forceinline__ int bin_s(int room, int s_group) { return max(1, min(room, s_group)); }

/* The plan from the counts, in one block: what plan_group_eval and GroupLaunch::plan compute on the host.  Bins are
 * read in tiles of one bin per thread. */
__global__ void __launch_bounds__(kPlanThreads) group_plan_kernel(const GroupPlanParams p)
{
    typedef cub::BlockReduce<long long, kPlanThreads> Reduce;
    typedef cub::BlockScan<PlanSums, kPlanThreads> Scan;
    __shared__ union {
        typename Reduce::TempStorage reduce;
        typename Scan::TempStorage scan;
    } temp;
    __shared__ int s_group_s;
    __shared__ long long per_unit_s;
    const int tid = threadIdx.x;
    const int nbins = p.nbins;

    /* s_group: from s_start down to s_floor, the first s at which the launch has at least items_wanted items */
    if (tid == 0) s_group_s = p.s_start;
    if (p.shrink && p.s_start > p.s_floor) {
        long long items[kMaxShrink + 1];
#pragma unroll
        for (int t = 0; t <= kMaxShrink; t++) items[t] = 0;
        for (int g = tid; g < nbins; g += kPlanThreads) {
            const GroupBinInfo b = p.bin_info[g];
            const long long groups = (p.hist[g] + 31) / 32;
#pragma unroll
            for (int t = 1; t <= kMaxShrink; t++)
                items[t] += groups * (long long)((uint64_t)b.rows >> (min(b.room, t) + p.lane_bits));
        }
        __syncthreads();                  /* s_group_s is written */
        for (int t = p.s_start; t > p.s_floor; t--) {
            long long mine = 0;
#pragma unroll
            for (int u = 1; u <= kMaxShrink; u++)
                if (u == t) mine = items[u];
            const long long all = Reduce(temp.reduce).Sum(mine);
            if (tid == 0 && s_group_s == t && all < p.items_wanted) s_group_s = t - 1;
            __syncthreads();
        }
    }
    __syncthreads();
    const int s_group = s_group_s;

    /* work units: items per unit from every key group's items */
    if (tid == 0) per_unit_s = 1;
    if (p.units) {
        long long items = 0;
        for (int g = tid; g < nbins; g += kPlanThreads) {
            const GroupBinInfo b = p.bin_info[g];
            items += (long long)((p.hist[g] + 31) / 32) * (long long)((uint64_t)b.rows >> (bin_s(b.room, s_group) + p.lane_bits));
        }
        const long long all = Reduce(temp.reduce).Sum(items);
        if (tid == 0) per_unit_s = max(1ll, min((all + p.grid - 1) / p.grid, (long long)p.unit_cap));
    }
    __syncthreads();
    const long long per_unit = per_unit_s;

    /* every bin's first sorted key, key group and work unit: exclusive scans over the bins in order */
    PlanSums carry{0, 0, 0};
    for (int g0 = 0; g0 < nbins; g0 += kPlanThreads) {
        const int g = g0 + tid;
        PlanSums mine{0, 0, 0};
        int s = 0;
        if (g < nbins) {
            const GroupBinInfo b = p.bin_info[g];
            s = bin_s(b.room, s_group);
            mine.keys = p.hist[g];
            mine.groups = (mine.keys + 31) / 32;
            if (p.units) {
                const long long nsub = (long long)((uint64_t)b.rows >> (s + p.lane_bits));
                mine.units = mine.groups * ((nsub + per_unit - 1) / per_unit);
            }
        }
        PlanSums first, tile;
        Scan(temp.scan).ExclusiveScan(mine, first, PlanSums{0, 0, 0}, PlanAdd(), tile);
        if (g < nbins)
            p.bin_first[g] = make_uint4((uint32_t)(carry.keys + first.keys), (uint32_t)(carry.groups + first.groups),
                                        (uint32_t)(carry.units + first.units), (uint32_t)s);
        carry = PlanAdd()(carry, tile);
        __syncthreads();                  /* temp.scan is reused */
    }
    if (tid == 0) {
        p.counts[0] = (uint32_t)carry.groups;
        p.counts[1] = (uint32_t)carry.units;
        p.counts[2] = p.hist[nbins];
        p.counts[3] = (uint32_t)per_unit;
        if (p.bad) *p.bad = (int64_t)p.hist[nbins];
    }
}

/* The last bin whose first entry (bin_first[g].y, or .z with `units`) is <= i: the bin of key group or work unit i,
 * as bins without any have the first entry of the next bin */
__device__ __forceinline__ int bin_of(const uint4 *bin_first, int nbins, uint32_t i, bool units)
{
    int lo = 0, hi = nbins;               /* the answer is in [lo, hi) */
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        const uint32_t f = units ? bin_first[mid].z : bin_first[mid].y;
        if (f <= i) lo = mid;
        else hi = mid;
    }
    return lo;
}

/* descs[k] for every key group k and, with `units`, units[u] for every work unit u: the entries GroupLaunch::plan
 * writes.  Key group j of bin g holds its sorted keys 32 j .. 32 j + 31; a group of nsub items is cut into
 * ceil(nsub / per_unit) units, unit i holding items nsub i / parts .. nsub (i + 1) / parts. */
__global__ void __launch_bounds__(256) group_emit_kernel(const GroupPlanParams p)
{
    const uint32_t ngroups = p.counts[0], nunits = p.counts[1], per_unit = p.counts[3];
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < ngroups; k += stride) {
        const int g = bin_of(p.bin_first, p.nbins, k, false);
        const uint4 f = p.bin_first[g];
        const GroupBinInfo b = p.bin_info[g];
        const uint32_t j = k - f.y, count = p.hist[g];
        GroupDesc d;
        d.key_first = f.x + 32u * j;
        d.nkeys = min(32u, count - 32u * j);
        d.depth = b.depth;
        d.s = (int32_t)f.w;
        d.nsub = (uint32_t)((uint64_t)b.rows >> (f.w + (uint32_t)p.lane_bits));
        d.pad = 0;
        d.table_off_v = b.table_off_v;
        p.descs[k] = d;
    }
    if (!p.units) return;
    for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < nunits; u += stride) {
        const int g = bin_of(p.bin_first, p.nbins, u, true);
        const uint4 f = p.bin_first[g];
        const uint64_t nsub = (uint64_t)p.bin_info[g].rows >> (f.w + (uint32_t)p.lane_bits);
        const uint32_t parts = (uint32_t)((nsub + per_unit - 1) / per_unit);
        const uint32_t r = u - f.z, j = r / parts, i = r - j * parts;
        const uint64_t first = nsub * i / parts, end = nsub * (i + 1) / parts;
        p.units_out[u] = WorkUnit{f.y + j, (uint32_t)first, (uint32_t)(end - first), 0u};
    }
}

int grid_for(int64_t work, int per_block, int sm_count)
{
    const int64_t cap = (int64_t)(sm_count > 0 ? sm_count : 1) * 8;
    const int64_t blocks = (work + per_block - 1) / per_block;
    return (int)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

}  // namespace

cudaError_t group_plan_temp_bytes(int64_t nkeys, int end_bit, size_t *bytes)
{
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                           (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)nkeys, 0, end_bit);
}

cudaError_t launch_group_plan(const GroupPlanParams &p, int sm_count, cudaStream_t stream)
{
    cudaError_t e = cudaMemsetAsync(p.hist, 0, ((size_t)p.nbins + 1) * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    group_hist_kernel<<<grid_for(p.nkeys, 256, sm_count), 256, 0, stream>>>(p.bins, p.nkeys, p.nbins, p.hist, p.keys_in,
                                                                           p.vals_in);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    size_t temp_bytes = p.temp_bytes;
    e = cub::DeviceRadixSort::SortPairs(p.temp, temp_bytes, p.keys_in, p.keys_out, p.vals_in, p.vals_out, (int)p.nkeys, 0,
                                        p.end_bit, stream);
    if (e != cudaSuccess) return e;
    group_order_kernel<<<grid_for(p.nkeys, 256, sm_count), 256, 0, stream>>>(p.keys_out, p.vals_out, p.nkeys, p.nbins,
                                                                            p.bin_info, p.order);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    group_plan_kernel<<<1, kPlanThreads, 0, stream>>>(p);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    group_emit_kernel<<<grid_for(p.descs_cap + (p.units ? p.units_cap : 0), 256, sm_count), 256, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace b200dpf
