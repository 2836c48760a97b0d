/*
 * dpf_kernels.cu -- sm_90a kernels of the DPF evaluation engine.
 *
 * One kernel does the whole hot path of the reference's dpf_hybrid_kernel
 * (dpf_gpu/dpf/dpf_hybrid.cu:38-256): GGM-tree expansion of every key over the
 * full domain, fused with the inner product against the table, plus the
 * reduction -- but organised for Hopper rather than translated:
 *
 *   work item   = (group of 32 keys) x (one 2^s-leaf subtree).  A warp owns a
 *                 work item; LANE = KEY.  All 32 lanes walk the same tree shape,
 *                 so control flow is warp-uniform and every table row a warp
 *                 needs is ONE broadcast 128-bit load shared by 32 keys (the
 *                 reference re-reads the table once per key).  For batches
 *                 smaller than a warp the mapping generalises to lane = (key,
 *                 subtree slot): kpw keys x 32/kpw adjacent subtrees per warp, so a
 *                 single query still uses every lane (the role the reference gives
 *                 to dpf_coop.cu).
 *   expansion   = per-thread depth-first search: a node's two children are
 *                 produced together in registers (shared AES key schedule /
 *                 shared first-round quarter rounds), the right child parks in a
 *                 per-thread shared-memory slot (one slot per tree height), the
 *                 left child is descended into; below height 2 the right child
 *                 waits in registers instead.  No global scratch, no
 *                 __syncthreads in the main loop (the reference ping-pongs two
 *                 global stacks with two barriers per step).
 *   MAC         = only the low 32 bits of a leaf survive (dpf_wrapper.cu:182),
 *                 so the product is 32-bit IMADs against an int32 table stored
 *                 in breadth-first leaf order (4x less table traffic than the
 *                 reference's 128-bit table, ~20x fewer MAC instructions).
 *   corrections = the 32 keys' correction words live in shared memory, laid out
 *                 [level][bank][bit][key] so a warp's 16-byte reads are
 *                 conflict free.
 *   AES         = T-table AES with the four tables replicated per bank in
 *                 shared memory (4 x 32 KiB): lane L only ever touches bank L,
 *                 so lookups are conflict-free, and the shared address of a
 *                 lookup is formed by ONE PRMT (byte insert into a 64 KiB-aligned
 *                 base) + the LDS immediate offset.
 *   frontier    = the top of every key's tree is expanded once and the seeds of all
 *                 depth-F nodes stored; work items then start from their frontier
 *                 node instead of re-walking from the root, so items can be small
 *                 (good load balance) without paying a root-to-subtree walk each.
 *   one launch  = a whole evaluation is ONE cooperative launch: phase `top` clears the
 *                 result and the ticket counters and builds the frontier, a grid-wide
 *                 barrier follows, phase `main` does the work and block 0 re-arms the
 *                 top-phase tickets for the next launch.  (The reference's step is
 *                 cudaMemcpy + kernel + cudaMemcpy with a stream created per call,
 *                 dpf_wrapper.cu:150-176; ours was memset, memset, kernel, kernel.)
 *   wide rows   = NV uint4 of a table row per pass (16/32/64 int32 columns): the
 *                 first 64 bytes of both rows are prefetched before the leaf
 *                 expansion, the rest streamed chunk by chunk during the MAC.
 *   scheduling  = persistent blocks; warps draw subtrees from a per-key-group
 *                 ticket counter (atomicAdd), blocks migrate to the next key
 *                 group when theirs runs dry, partial sums leave through
 *                 red.global.add.u32.
 */
#include "dpf_kernels.cuh"

#include <algorithm>
#include <atomic>

#include <cub/device/device_radix_sort.cuh>

#include "dpf_core.cuh"

namespace b200dpf {

namespace {

__constant__ uint32_t c_te0[256];

/* ---- AES table policy on the device -------------------------------------- */
struct AesSmemTables {
    /* shared-window address of (table region + lane*4); the region base is a
     * multiple of 64 KiB, so byte 1 of this value is zero. */
    uint32_t lanebase;

    template <int K, int BYTE>
    __device__ __forceinline__ uint32_t te(uint32_t word) const
    {
        /* address = lanebase with byte 1 replaced by the index byte:
         * entry v of table K for lane L sits at v*256 + (K&1)*128 + (K>>1)*65536 + L*4 */
        const uint32_t addr = __byte_perm(word, lanebase, 0x7604u | (BYTE << 4));
        uint32_t v;
        asm("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"((K & 1) * 128 + (K >> 1) * 65536));
        return v;
    }
};

struct NoTables {
    template <int K, int BYTE>
    __device__ __forceinline__ uint32_t te(uint32_t) const { return 0; }
};

template <int PRF> struct TablePolicy { typedef NoTables type; };
template <> struct TablePolicy<PRF_AES128> { typedef AesSmemTables type; };

/* ---- cp.async.bulk (TMA) + mbarrier primitives ----------------------------- */
namespace tma {

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t done = 0;
    for (uint32_t spin = 0; !done; spin++) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (spin > (1u << 28)) __trap();   /* a lost arrival must not hang the GPU */
    }
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

}  // namespace tma

/* ---- per-thread environment for the shared traversal code ---------------- */
template <int PRF, int NV, int THREADS, int MODE>
struct DevEnv {
    typename TablePolicy<PRF>::type ta;
    const uint4 *cw_lane;       /* &cw_s[lane]; entry (level,bank,bit) at +((level*2+bank)*2+bit)*32 */
    const uint32_t *cwlo_lane;  /* &cwlo_s[lane]; entry (bank,bit) at +(bank*2+bit)*32 */
    uint4 *stack_lo, *stack_hi; /* pre-offset by tid; level l at +l*THREADS */
    int stack_split;
    const uint4 *rows;          /* first row of the current subtree, at this pass's column */
    uint32_t row_stride_v;
    uint32_t acc[4 * NV];
    uint4 ra[4], rb[4];         /* prefetched first 64 bytes of the two rows of a leaf pair */
    uint32_t *leaf_out;         /* leaf cache slot of the subtree's first leaf for this lane, or null */
    uint4 *front_out;           /* MODE_FRONTIER: &frontier[(kg*nfront + first node)*kpw + key slot] */
    uint32_t kpw;               /* keys per warp */
    /* expand mode */
    uint32_t *share_row;        /* shares + key*n */
    uint32_t pos_base;          /* global leaf position of the subtree's first leaf */
    int depth;
    bool key_valid;

    __device__ __forceinline__ Seed cw(int level, uint32_t bank, uint32_t bit) const
    {
        const uint4 v = cw_lane[((level * 2 + (int)bank) * 2 + (int)bit) * 32];
        return make_seed(v.x, v.y, v.z, v.w);
    }
    __device__ __forceinline__ uint32_t cw_lo(uint32_t bank, uint32_t bit) const
    {
        return cwlo_lane[(bank * 2 + bit) * 32];
    }
    __device__ __forceinline__ uint4 *slot(int h) const
    {
        const int l = h - 1;
        return (l < stack_split ? stack_lo : stack_hi) + l * THREADS;
    }
    __device__ __forceinline__ void push(int h, const Seed &s) const
    {
        *slot(h) = make_uint4(s.x, s.y, s.z, s.w);
    }
    __device__ __forceinline__ Seed pop(int h) const
    {
        const uint4 v = *slot(h);
        return make_seed(v.x, v.y, v.z, v.w);
    }
    static constexpr ModeTraits M = mode_traits(MODE);
    /* early-terminated keys (four rows per leaf) prefetch the first row pair before the leaf expansion
     * at 16 columns only: at 32, rows held across the full-width expansion (or two rows in flight
     * beside the next two) spill */
    static constexpr bool ET_PREFETCH = M.result == RESULT_ADD && M.row_shift != 0 && NV == 4;
    /* ROWS_STAGED: the work item's 2^s rows were requested with one cp.async.bulk when the item was
     * drawn; they are first needed s-1 node expansions later, which hides the copy */
    const uint4 *tile;          /* this warp's staged rows (shared memory) */
    uint32_t tile_bar;          /* shared-window address of this warp's mbarrier */
    uint32_t tile_phase;
    bool tile_pending;

    __device__ __forceinline__ void leaf_prefetch(uint32_t local_pos)
    {
        if (M.result == RESULT_XOR) {
            /* 256 rows per leaf pair: leaf_bits streams them */
        } else if (M.row_load == ROWS_STAGED) {
            if (tile_pending) {
                tma::mbar_wait(tile_bar, tile_phase);
                tile_phase ^= 1u;
                tile_pending = false;
            }
            const uint4 *r = tile + (size_t)local_pos * 4;
#pragma unroll
            for (int j = 0; j < 4; j++) ra[j] = r[j];
#pragma unroll
            for (int j = 0; j < 4; j++) rb[j] = r[4 + j];
        } else if (M.row_load == ROWS_COLSPLIT) {
            ra[0] = __ldg(rows + (size_t)local_pos * row_stride_v);
            rb[0] = __ldg(rows + (size_t)(local_pos + 1) * row_stride_v);
        } else if (M.feeds == FEEDS_MAC && ET_PREFETCH) {
            /* the first 64 bytes of the two rows multiplied first: lane 0 of both leaves */
            const uint4 *r = rows + (size_t)local_pos * 4 * row_stride_v;
#pragma unroll
            for (int j = 0; j < 4; j++) ra[j] = __ldg(r + j);
#pragma unroll
            for (int j = 0; j < 4; j++) rb[j] = __ldg(r + 4 * row_stride_v + j);
        } else if (M.feeds == FEEDS_MAC && M.row_shift == 0) {
            const uint4 *r = rows + (size_t)local_pos * row_stride_v;
#pragma unroll
            for (int j = 0; j < 4; j++) ra[j] = __ldg(r + j);
#pragma unroll
            for (int j = 0; j < 4; j++) rb[j] = __ldg(r + row_stride_v + j);
        }
    }
    /* early-terminated keys: leaves local_pos and local_pos + 1 with their four row shares each, against
     * rows 4 local_pos .. 4 local_pos + 7 */
    /* XOR-shared keys: leaves local_pos and local_pos + 1 with 128 share bits each, against rows 128 local_pos
     * .. 128 local_pos + 255.  Column split: rows points at this lane's 16 bytes of the row (columns 4 (lane & 3)
     * .. +3), and acc[4 j + c] is column 4 (lane & 3) + c of key kslot ^ j, whose leaf words come from lane ^ j
     * by SHFL, one word (32 rows) at a time.  A row costs each lane one 16-byte load and, per key, a mask
     * from its share bit and 4 LOP3 (acc ^= row & mask).  Correct only when the four lanes of a quad hold
     * four different keys at the same leaf position (kpw >= 4): launch_eval refuses a column-split launch
     * with kpw_log2 < 2. */
    __device__ __forceinline__ void leaf_bits(uint32_t local_pos, const Seed &w0, const Seed &w1)
    {
        uint32_t w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};   /* word k: rows 32 k .. 32 k + 31 */
        const uint4 *r = rows + (size_t)local_pos * 128 * row_stride_v;
#pragma unroll 1
        for (int k = 0; k < 8; k++) {
            uint32_t u[4];
            u[0] = w[0];
#pragma unroll
            for (int j = 1; j < 4; j++) u[j] = __shfl_xor_sync(0xffffffffu, w[0], j);
#pragma unroll
            for (int i = 0; i < 7; i++) w[i] = w[i + 1];
#pragma unroll 1
            for (int b0 = 0; b0 < 32; b0 += 8) {
                uint4 t[8];   /* eight rows in flight */
#pragma unroll
                for (int i = 0; i < 8; i++) t[i] = __ldg(r + (size_t)i * row_stride_v);
#pragma unroll
                for (int i = 0; i < 8; i++) {
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const uint32_t m = (uint32_t)((int32_t)(u[j] << (31 - i)) >> 31);   /* bit b0 + i */
                        acc[4 * j + 0] ^= t[i].x & m;
                        acc[4 * j + 1] ^= t[i].y & m;
                        acc[4 * j + 2] ^= t[i].z & m;
                        acc[4 * j + 3] ^= t[i].w & m;
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; j++) u[j] >>= 8;
                r += (size_t)8 * row_stride_v;
            }
        }
    }
    __device__ __forceinline__ void leaf_quads(uint32_t local_pos, const Seed &w0, const Seed &w1)
    {
        if constexpr (M.feeds == FEEDS_MAC && M.result == RESULT_XOR) {
            leaf_bits(local_pos, w0, w1);
            return;
        }
        const uint32_t a[4] = {w0.x, w0.y, w0.z, w0.w}, b[4] = {w1.x, w1.y, w1.z, w1.w};
        if (M.feeds == FEEDS_MAC) {
            if (leaf_out != nullptr) {   /* coalesced: 32 keys x 4 bytes per row */
#pragma unroll
                for (int l = 0; l < 4; l++) {
                    leaf_out[((size_t)local_pos * 4 + l) * 32] = a[l];
                    leaf_out[((size_t)local_pos * 4 + 4 + l) * 32] = b[l];
                }
            }
            const uint4 *r0 = rows + (size_t)local_pos * 4 * row_stride_v;
            if constexpr (ET_PREFETCH) {
                /* 16 columns: rows in pairs (4 local_pos + l, 4 local_pos + 4 + l), the first pair prefetched
                 * by leaf_prefetch, the next pair's loads issued before the current one is multiplied */
#pragma unroll
                for (int l = 0; l < 4; l++) {
                    uint4 na[4], nb[4];
                    if (l + 1 < 4) {
                        const uint4 *r = r0 + (size_t)(l + 1) * row_stride_v;
#pragma unroll
                        for (int j = 0; j < 4; j++) na[j] = __ldg(r + j);
#pragma unroll
                        for (int j = 0; j < 4; j++) nb[j] = __ldg(r + 4 * row_stride_v + j);
                    }
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        acc[4 * j + 0] += a[l] * ra[j].x + b[l] * rb[j].x;
                        acc[4 * j + 1] += a[l] * ra[j].y + b[l] * rb[j].y;
                        acc[4 * j + 2] += a[l] * ra[j].z + b[l] * rb[j].z;
                        acc[4 * j + 3] += a[l] * ra[j].w + b[l] * rb[j].w;
                    }
                    if (l + 1 < 4) {
#pragma unroll
                        for (int j = 0; j < 4; j++) { ra[j] = na[j]; rb[j] = nb[j]; }
                    }
                }
            } else {
                /* 32 columns: one whole row per step, the row loop kept rolled (unrolled, the compiler
                 * hoists the loads of several rows and spills) */
#pragma unroll 1
                for (int row = 0; row < 8; row++) {
                    const uint4 *r = r0 + (size_t)row * row_stride_v;
                    uint4 t[NV];
#pragma unroll
                    for (int j = 0; j < NV; j++) t[j] = __ldg(r + j);
                    const uint32_t v = row == 0 ? a[0] : row == 1 ? a[1] : row == 2 ? a[2] : row == 3 ? a[3]
                                     : row == 4 ? b[0] : row == 5 ? b[1] : row == 6 ? b[2] : b[3];
#pragma unroll
                    for (int j = 0; j < NV; j++) {
                        acc[4 * j + 0] += v * t[j].x;
                        acc[4 * j + 1] += v * t[j].y;
                        acc[4 * j + 2] += v * t[j].z;
                        acc[4 * j + 3] += v * t[j].w;
                    }
                }
            }
        } else if (M.feeds == FEEDS_SHARES && key_valid) {
            /* leaf position p holds leaf bitrev_depth(p), whose word l is the share of row 4 * leaf + l */
            const uint32_t p = pos_base + local_pos;
            uint32_t *o0 = share_row + 4 * (size_t)(__brev(p) >> (32 - depth));
            uint32_t *o1 = share_row + 4 * (size_t)(__brev(p + 1) >> (32 - depth));
#pragma unroll
            for (int l = 0; l < 4; l++) {   /* the caller's buffer need not be 16-byte aligned */
                o0[l] = a[l];
                o1[l] = b[l];
            }
        }
    }
    __device__ __forceinline__ void leaf_pair(uint32_t local_pos, uint32_t v0, uint32_t v1)
    {
        if (M.feeds == FEEDS_MAC) {
            if (leaf_out != nullptr) {   /* coalesced: 32 keys x 4 bytes per leaf */
                leaf_out[(size_t)local_pos * 32] = v0;
                leaf_out[(size_t)(local_pos + 1) * 32] = v1;
            }
            if constexpr (M.row_load == ROWS_COLSPLIT) {
                /* rows points at this lane's 16 bytes of the row; acc[4 j + c] is column 4 (lane & 3) + c of
                 * key kslot ^ j, whose leaf values come from lane ^ j */
                uint32_t u0[4], u1[4];
                u0[0] = v0;
                u1[0] = v1;
#pragma unroll
                for (int j = 1; j < 4; j++) {
                    u0[j] = __shfl_xor_sync(0xffffffffu, v0, j);
                    u1[j] = __shfl_xor_sync(0xffffffffu, v1, j);
                }
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    acc[4 * j + 0] += u0[j] * ra[0].x + u1[j] * rb[0].x;
                    acc[4 * j + 1] += u0[j] * ra[0].y + u1[j] * rb[0].y;
                    acc[4 * j + 2] += u0[j] * ra[0].z + u1[j] * rb[0].z;
                    acc[4 * j + 3] += u0[j] * ra[0].w + u1[j] * rb[0].w;
                }
                return;
            }
            const uint4 *r = rows + (size_t)local_pos * row_stride_v;
#pragma unroll
            for (int c = 0; c < NV / 4; c++) {
                uint4 na[4], nb[4];
                if (c + 1 < NV / 4) {   /* next 64 bytes of both rows while this chunk is multiplied */
#pragma unroll
                    for (int j = 0; j < 4; j++) na[j] = __ldg(r + 4 * (c + 1) + j);
#pragma unroll
                    for (int j = 0; j < 4; j++) nb[j] = __ldg(r + row_stride_v + 4 * (c + 1) + j);
                }
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    acc[16 * c + 4 * j + 0] += v0 * ra[j].x + v1 * rb[j].x;
                    acc[16 * c + 4 * j + 1] += v0 * ra[j].y + v1 * rb[j].y;
                    acc[16 * c + 4 * j + 2] += v0 * ra[j].z + v1 * rb[j].z;
                    acc[16 * c + 4 * j + 3] += v0 * ra[j].w + v1 * rb[j].w;
                }
                if (c + 1 < NV / 4) {
#pragma unroll
                    for (int j = 0; j < 4; j++) { ra[j] = na[j]; rb[j] = nb[j]; }
                }
            }
        } else if (M.feeds == FEEDS_SHARES && key_valid) {
            /* leaf position p holds index bitrev_depth(p) */
            const uint32_t p = pos_base + local_pos;
            share_row[__brev(p) >> (32 - depth)] = v0;
            share_row[__brev(p + 1) >> (32 - depth)] = v1;
        }
    }
    /* FEEDS_FRONTIER: whole seeds of two adjacent frontier nodes */
    __device__ __forceinline__ void node_pair(uint32_t local_pos, const Seed &c0, const Seed &c1)
    {
        front_out[(size_t)local_pos * kpw] = make_uint4(c0.x, c0.y, c0.z, c0.w);
        front_out[(size_t)(local_pos + 1) * kpw] = make_uint4(c1.x, c1.y, c1.z, c1.w);
    }
};

extern __shared__ __align__(16) unsigned char g_dyn_smem[];

/* Grid-wide barrier of a cooperative launch (every block is resident, so spinning cannot
 * deadlock).  `bar` only ever counts up; `target` is the value it has once every block of THIS
 * launch has arrived (the host keeps the running total), compared wrap-safe. */
__device__ __forceinline__ void grid_barrier(uint32_t *bar, uint32_t target)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(bar, 1u);
        for (uint32_t spin = 0;; spin++) {
            uint32_t v;
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
            if ((int32_t)(v - target) >= 0) break;
            if (spin > (1u << 25)) __trap();   /* a lost arrival must not hang the GPU */
            __nanosleep(40);
        }
        __threadfence();
    }
    __syncthreads();
}

/* One traversal phase of a launch: every block walks the key groups (starting at its own offset so
 * blocks spread over groups), loads a group's correction words into shared memory when the group
 * still has tickets, and its warps draw work items until the group runs dry. */
__device__ __forceinline__ unsigned long long global_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

/* The correction words of the kpw keys of a key group -> shared, [level][bank][bit][key], and their root
 * seeds; keys past `key_last` load key_last's words */
template <int THREADS>
__device__ __forceinline__ void load_key_group(const EvalParams &p, int depth, int key_first, int key_last, int kpw,
                                               uint4 *cw_s, uint32_t *cwlo_s, uint4 *root_s)
{
    const int tid = threadIdx.x;
    const int per_key = depth * 4;
    for (int i = tid; i < per_key * kpw; i += THREADS) {
        const int k = i / per_key;            /* key within the group   */
        const int e = i - k * per_key;        /* (bank, level, bit)     */
        const int bank = e / (depth * 2);
        const int lb = e - bank * (depth * 2);     /* 2*level + bit       */
        int key = key_first + k;
        if (key > key_last) key = key_last;
        const int level = lb >> 1, bit = lb & 1;
        const uint32_t slot = p.key_compact ? 2u + 4u * (uint32_t)level + 2u * (uint32_t)bank + (uint32_t)bit
                                            : (bank ? 65u : 1u) + (uint32_t)lb;
        const uint4 v = __ldg(p.keys + (size_t)key * p.key_stride_v + slot);
        cw_s[((level * 2 + bank) * 2 + bit) * 32 + k] = v;
        if (level == 0) cwlo_s[(bank * 2 + bit) * 32 + k] = v.x;
    }
    if (tid < kpw) {
        int key = key_first + tid;
        if (key > key_last) key = key_last;
        root_s[tid] = __ldg(p.keys + (size_t)key * p.key_stride_v + p.key_root_v);
    }
}

/* `quota`: tickets this WARP may draw in this call over all key groups (0xffffffff = no limit). */
template <int PRF, int NV, int THREADS, int MODE>
__device__ __forceinline__ void run_phase(const EvalParams &p, const PhaseParams &ph,
                                          const typename TablePolicy<PRF>::type &ta, uint32_t quota = 0xffffffffu)
{
    constexpr ModeTraits M = mode_traits(MODE);
    const int tid = threadIdx.x;
    const int lane = tid & 31;

    uint4 *cw_s = reinterpret_cast<uint4 *>(g_dyn_smem + p.off_cw);
    uint32_t *cwlo_s = reinterpret_cast<uint32_t *>(g_dyn_smem + p.off_cwlo);
    uint4 *root_s = reinterpret_cast<uint4 *>(g_dyn_smem + p.off_root);
    volatile int *flag_s = reinterpret_cast<volatile int *>(g_dyn_smem + p.off_flag);

    /* lane -> (key slot within the group, subtree slot within the ticket) */
    const int kpw = 1 << p.kpw_log2;
    const int spw_log2 = 5 - p.kpw_log2;
    const int kslot = lane & (kpw - 1);
    const uint32_t sslot = (uint32_t)lane >> p.kpw_log2;
    const uint32_t ntickets = ph.nsub >> spw_log2;

    DevEnv<PRF, NV, THREADS, MODE> env;
    env.ta = ta;
    env.cw_lane = cw_s + kslot;
    env.cwlo_lane = cwlo_s + kslot;
    env.kpw = (uint32_t)kpw;
    env.stack_lo = reinterpret_cast<uint4 *>(g_dyn_smem + p.off_stack_lo) + tid;
    env.stack_hi = reinterpret_cast<uint4 *>(g_dyn_smem + p.off_stack_hi) + tid - ph.stack_split * THREADS;
    env.stack_split = ph.stack_split;
    env.row_stride_v = p.row_stride_v;
    env.depth = p.depth;
    if constexpr (M.row_load == ROWS_STAGED) {
        const int w = tid >> 5;
        env.tile = reinterpret_cast<const uint4 *>(g_dyn_smem + p.off_tile + ((size_t)w << (ph.s + 6)));
        env.tile_bar = (uint32_t)__cvta_generic_to_shared(g_dyn_smem + p.off_tile_bar + 8 * w);
        env.tile_phase = 0;
        env.tile_pending = false;
        if (lane == 0) {
            tma::mbar_init(env.tile_bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }

    uint32_t taken = 0;
    /* the key groups: those the device planned (read once), or p.key_groups */
    int dev_groups = 0;
    if constexpr (M.counts_on_device) dev_groups = (int)p.dev_counts[0];
    auto key_groups = [&]() { return M.counts_on_device ? dev_groups : p.key_groups; };
    for (int j = 0; j < key_groups(); j++) {
        const int kg = (int)((blockIdx.x + (unsigned)j) % (unsigned)key_groups());

        /* what this key group evaluates: the context's one table, or (grouped) its own bin */
        int g_depth = p.depth, g_s = ph.s, g_walk_first = ph.walk_first_level, g_walk_steps = ph.walk_steps;
        int g_key_first = kg * kpw, g_key_last = p.nkeys - 1;
        uint32_t g_tickets = ntickets;
        const uint4 *g_table = p.table;
        if (M.grouped) {
            const GroupDesc g = p.groups[kg];
            g_depth = g.depth;
            g_s = g.s;
            g_walk_first = g.depth - 1;
            g_walk_steps = g.depth - g.s;
            g_key_first = (int)g.key_first;
            g_key_last = (int)(g.key_first + g.nkeys) - 1;
            g_tickets = g.nsub;
            g_table = p.table + g.table_off_v;
        }

        if (quota != 0xffffffffu && __syncthreads_and(taken >= quota)) break;   /* the block's share is done */
        if (tid == 0) *flag_s = (*reinterpret_cast<volatile uint32_t *>(ph.counters + kg) < g_tickets) ? 1 : 0;
        __syncthreads();
        const bool has_work = (*flag_s != 0);
        if (has_work) load_key_group<THREADS>(p, g_depth, g_key_first, g_key_last, kpw, cw_s, cwlo_s, root_s);
        __syncthreads();
        if (!has_work) continue;

        const int key = g_key_first + kslot;
        env.key_valid = key <= g_key_last;
        if (M.feeds == FEEDS_MAC) {
#pragma unroll
            for (int e = 0; e < 4 * NV; e++) env.acc[e] = 0;
        } else if (M.feeds == FEEDS_SHARES) {
            /* XOR-shared keys: one bit per row, n / 32 words per key */
            env.share_row = p.shares + (size_t)(env.key_valid ? key : 0) * (M.result == RESULT_XOR ? p.n >> 5 : p.n);
        }
        const uint4 rv = root_s[kslot];
        const Seed root = make_seed(rv.x, rv.y, rv.z, rv.w);

        /* SMALL items (<= 15 node pairs) draw their tickets one draw ahead, so the atomic's round trip
         * to L2 overlaps the items being expanded instead of stalling the warp between items.  Big items
         * draw when they are done: holding a ticket for the length of a 127-pair item makes the hand-out
         * one item less adaptive at the end of a key group (slower at n = 2^20 when measured before the
         * H100 port), and the atomic's latency is nothing against it.
         * A draw takes a CHUNK of consecutive items, sized from what is left: (remaining / 8x the
         * warps of the grid), between 1 and 8 -- guided self-scheduling: big early chunks when a key
         * group holds many more items than the grid has warps, single items at the end keep the tail
         * fine-grained.  (Cutting a group's tickets into several counters was tried for the case of
         * one or two key groups per GPU and measured slower.) */
        const uint32_t grid_warps = gridDim.x * (uint32_t)(THREADS / 32);
        const bool chunked = quota == 0xffffffffu;          /* the balanced top round counts single tickets */
        const bool ahead = g_s <= 4;
        uint32_t chunk = 1;
        if (chunked) chunk = min(8u, max(1u, g_tickets / (8u * grid_warps)));
        uint32_t t_raw = 0;
        bool draw = taken < quota;
        if (draw && lane == 0) t_raw = atomicAdd(ph.counters + kg, chunk);
        while (draw) {
            const uint32_t t0 = __shfl_sync(0xffffffffu, t_raw, 0);
            if (t0 >= g_tickets) break;
            const uint32_t t1 = min(t0 + chunk, g_tickets);
            taken += t1 - t0;
            draw = taken < quota;
            if (chunked) chunk = min(8u, max(1u, (g_tickets - t1) / (8u * grid_warps)));
            if (ahead && draw && lane == 0) t_raw = atomicAdd(ph.counters + kg, chunk);
          for (uint32_t t = t0; t < t1; t++) {
            const uint32_t q = (t << spw_log2) + sslot;   /* this lane's subtree */
            Seed start = root;
            if (ph.frontier_in != nullptr) {
                /* written earlier in this launch (before the grid barrier) or by the previous one:
                 * read through L2, never a stale L1 line */
                const uint4 fv = __ldcg(ph.frontier_in + ((size_t)kg * p.nfront + (q >> ph.front_shift)) * kpw + kslot);
                start = make_seed(fv.x, fv.y, fv.z, fv.w);
            }
            const Seed r = walk_down<PRF>(env, start, g_walk_first, g_walk_steps, ph.sub_first + q);
            if (M.feeds == FEEDS_FRONTIER) {
                env.front_out = p.frontier_out + ((size_t)kg * p.nfront + ((size_t)q << g_s)) * kpw + kslot;
                eval_subtree<PRF, true>(env, r, g_s, ph.level_base);
            } else {
                env.rows = g_table + ((size_t)q << (g_s + M.row_shift)) * p.row_stride_v + p.col_off_v +
                           (M.row_load == ROWS_COLSPLIT ? (lane & 3) : 0);
                if constexpr (M.row_load == ROWS_STAGED) {
                    /* the item's rows are one contiguous run (64-byte rows, breadth-first leaf order) */
                    __syncwarp();                                   /* every lane is done with the previous tile */
                    if (lane == 0) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        const uint32_t bytes = 64u << g_s;
                        tma::mbar_expect_tx(env.tile_bar, bytes);
                        tma::bulk_g2s((uint32_t)__cvta_generic_to_shared(const_cast<uint4 *>(env.tile)), env.rows, bytes, env.tile_bar);
                    }
                    env.tile_pending = true;
                }
                env.pos_base = (ph.sub_first + q) << g_s;
                env.leaf_out = (!M.grouped && p.leaf_cache)
                                   ? p.leaf_cache + ((size_t)kg * p.n_local + ((size_t)q << (g_s + M.row_shift))) * 32 + lane
                                   : nullptr;
                eval_subtree<PRF, false, decltype(env), mode_leaf_group(MODE)>(env, r, g_s, 0);
            }
          }
            if (!ahead && draw && lane == 0) t_raw = atomicAdd(ph.counters + kg, chunk);
        }

        if (M.feeds == FEEDS_MAC) {
            /* lanes that hold the same key (different subtree slots) fold their partial sums
             * first, so every key receives one red.add per warp and column, not 32/kpw */
            for (int off = kpw; off < 32; off <<= 1) {
#pragma unroll
                for (int e = 0; e < 4 * NV; e++) {
                    if constexpr (M.result == RESULT_XOR) env.acc[e] ^= __shfl_xor_sync(0xffffffffu, env.acc[e], off);
                    else env.acc[e] += __shfl_xor_sync(0xffffffffu, env.acc[e], off);
                }
            }
            if (M.row_load == ROWS_COLSPLIT) {
                if (sslot == 0) {
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int kj = g_key_first + (kslot ^ j);
                        if (kj > g_key_last) continue;
                        uint32_t *o = p.out + (size_t)kj * p.out_stride + p.col_off;
#pragma unroll
                        for (int c = 0; c < 4; c++) {
                            const uint32_t e = 4u * (uint32_t)(lane & 3) + (uint32_t)c;
                            if constexpr (M.result == RESULT_XOR) {
                                if (e < p.ncols) atomicXor(o + e, env.acc[4 * j + c]);
                            } else {
                                if (e < p.ncols) atomicAdd(o + e, env.acc[4 * j + c]);
                            }
                        }
                    }
                }
            } else if (env.key_valid && sslot == 0) {
                uint32_t *o = p.out + (size_t)key * p.out_stride + p.col_off;
#pragma unroll
                for (int e = 0; e < 4 * NV; e++)
                    if ((uint32_t)e < p.ncols) atomicAdd(o + e, env.acc[e]);
            }
        }
        __syncthreads();   /* everyone done with this group's correction words */
    }
}

/* The main phase of a mode that draws work units (ModeTraits::units: grouped, one key group = 32 keys of one
 * bin, column split).  run_phase makes every block visit every key group -- a counter read and two barriers
 * each, about 3.7 us per group (DESIGN.md section 9) -- which would be most of the time of XOR-shared keys.
 * Here thread 0 draws the block's next unit of the host's list; the block loads correction words and roots
 * only when the unit's key group is not the one already in shared memory, and its warps split the unit's
 * items.  Each unit ends with the flush of the accumulators: XOR is associative, so a flush per unit is
 * exact.  A block reads nothing of a key group it draws no unit of. */
template <int PRF, int NV, int THREADS, int MODE>
__device__ __forceinline__ void run_units(const EvalParams &p, const PhaseParams &ph, const typename TablePolicy<PRF>::type &ta)
{
    constexpr ModeTraits M = mode_traits(MODE);
    static_assert(M.grouped && M.feeds == FEEDS_MAC && M.row_load == ROWS_COLSPLIT && M.result == RESULT_XOR,
                  "work units: grouped column-split XOR evaluation only");
    constexpr uint32_t NW = THREADS / 32;
    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const uint32_t warp = (uint32_t)tid >> 5;

    uint4 *cw_s = reinterpret_cast<uint4 *>(g_dyn_smem + p.off_cw);
    uint32_t *cwlo_s = reinterpret_cast<uint32_t *>(g_dyn_smem + p.off_cwlo);
    uint4 *root_s = reinterpret_cast<uint4 *>(g_dyn_smem + p.off_root);
    volatile uint32_t *draw_s = reinterpret_cast<volatile uint32_t *>(g_dyn_smem + p.off_flag);   /* 2 slots */

    DevEnv<PRF, NV, THREADS, MODE> env;   /* lane = key: 32 keys per warp, one subtree slot */
    env.ta = ta;
    env.cw_lane = cw_s + lane;
    env.cwlo_lane = cwlo_s + lane;
    env.kpw = 32;
    env.stack_lo = reinterpret_cast<uint4 *>(g_dyn_smem + p.off_stack_lo) + tid;
    env.stack_hi = reinterpret_cast<uint4 *>(g_dyn_smem + p.off_stack_hi) + tid - ph.stack_split * THREADS;
    env.stack_split = ph.stack_split;
    env.row_stride_v = p.row_stride_v;
    env.depth = p.depth;
    env.leaf_out = nullptr;
    env.key_valid = true;

    uint32_t dev_units = 0;
    if constexpr (M.counts_on_device) dev_units = p.dev_counts[1];
    uint32_t loaded = 0xffffffffu;        /* the key group in shared memory (block-uniform) */
    for (uint32_t i = 0;; i++) {
        /* the two slots take turns: slot i & 1 is written again at draw i + 2, and every thread has read it
         * before it passes the barrier of draw i + 1 */
        if (tid == 0) draw_s[i & 1] = atomicAdd(ph.counters, 1u);
        __syncthreads();                  /* also: every warp is done with the previous unit */
        const uint32_t u = draw_s[i & 1];
        if (u >= (M.counts_on_device ? dev_units : p.nunits)) break;
        const WorkUnit unit = p.units[u];
        const GroupDesc g = p.groups[unit.group];
        const int key_first = (int)g.key_first, key_last = (int)(g.key_first + g.nkeys) - 1;
        if (unit.group != loaded) {
            load_key_group<THREADS>(p, g.depth, key_first, key_last, 32, cw_s, cwlo_s, root_s);
            __syncthreads();
            loaded = unit.group;
        }
        if (warp >= unit.count) continue;

        const uint4 rv = root_s[lane];
        const Seed root = make_seed(rv.x, rv.y, rv.z, rv.w);
#pragma unroll
        for (int e = 0; e < 4 * NV; e++) env.acc[e] = 0;
        const uint4 *table = p.table + g.table_off_v + p.col_off_v + (lane & 3);
        for (uint32_t q = unit.first + warp; q < unit.first + unit.count; q += NW) {
            const Seed r = walk_down<PRF>(env, root, g.depth - 1, g.depth - g.s, q);
            env.rows = table + ((size_t)q << (g.s + M.row_shift)) * p.row_stride_v;
            env.pos_base = q << g.s;
            eval_subtree<PRF, false, decltype(env), mode_leaf_group(MODE)>(env, r, g.s, 0);
        }
        /* acc[4 j + c] is column 4 (lane & 3) + c of key lane ^ j (DevEnv::leaf_bits) */
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int kj = key_first + (lane ^ j);
            if (kj > key_last) continue;
            uint32_t *o = p.out + (size_t)kj * p.out_stride + p.col_off;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const uint32_t e = 4u * (uint32_t)(lane & 3) + (uint32_t)c;
                if (e < p.ncols) atomicXor(o + e, env.acc[4 * j + c]);
            }
        }
    }
}

template <int PRF, int NV, int MODE>
__global__ void __launch_bounds__(eval_block_shape(PRF, NV, MODE).threads, eval_block_shape(PRF, NV, MODE).min_blocks)
dpf_eval_kernel(const __grid_constant__ EvalParams p)
{
    constexpr int THREADS = eval_block_shape(PRF, NV, MODE).threads;
    const int tid = threadIdx.x;
    unsigned long long *stamp = (p.timing != nullptr && tid == 0) ? p.timing + (size_t)blockIdx.x * 8 : nullptr;
    if (stamp) stamp[0] = global_ns();

    typename TablePolicy<PRF>::type ta;
    if constexpr (PRF == PRF_AES128) {
        /* replicate Te0..Te3 across the 32 banks: entry v, lane L */
        const uint32_t tab = (uint32_t)__cvta_generic_to_shared(g_dyn_smem + p.off_tab);
        if ((tab & 0xffffu) != 0) __trap();   /* layout contract with the host planner */
        for (int i = tid; i < 256 * 32; i += THREADS) {
            const uint32_t v = c_te0[i >> 5];
            unsigned char *e = g_dyn_smem + p.off_tab + (i >> 5) * 256 + (i & 31) * 4;
            *reinterpret_cast<uint32_t *>(e) = v;
            *reinterpret_cast<uint32_t *>(e + 128) = __funnelshift_l(v, v, 8);
            *reinterpret_cast<uint32_t *>(e + 65536) = __funnelshift_l(v, v, 16);
            *reinterpret_cast<uint32_t *>(e + 65536 + 128) = __funnelshift_l(v, v, 24);
        }
        ta.lanebase = tab + (tid & 31) * 4;
    }

    if constexpr (mode_traits(MODE).feeds != FEEDS_FRONTIER) {
        if (p.fuse_top) {
            /* single-launch pipeline: clear this launch's accumulators and main-phase tickets,
             * expand the top of every key's tree into the frontier, meet at the grid barrier */
            const uint64_t gtid = (uint64_t)blockIdx.x * THREADS + tid, gthreads = (uint64_t)gridDim.x * THREADS;
            for (uint64_t i = gtid; i < p.zero_a_words; i += gthreads) p.zero_a[i] = 0u;
            for (uint64_t i = gtid; i < p.zero_b_words; i += gthreads) p.zero_b[i] = 0u;
            if (stamp) stamp[1] = global_ns();
            if (p.top.nsub != 0) {
                /* round 1: every block takes its even share (warp w: quota/nwarps, +1 for the first
                 * quota%nwarps warps); round 2: whatever is left, first come first served */
                constexpr uint32_t NW = THREADS / 32;
                const uint32_t w = (uint32_t)tid >> 5;
                uint32_t bq = p.top_block_quota;
                const uint32_t kgs = (uint32_t)p.key_groups;
                if (bq != 0x7fffffffu && gridDim.x >= kgs) {
                    /* blocks start at key group blockIdx % key_groups: the nb blocks that start at a
                     * group share its tickets exactly, so round 1 leaves nothing behind */
                    const uint32_t nb = gridDim.x / kgs + ((blockIdx.x % kgs) < (gridDim.x % kgs) ? 1u : 0u);
                    const uint32_t tickets = p.top.nsub >> (5 - p.kpw_log2);
                    bq = (tickets + nb - 1) / nb;
                }
                run_phase<PRF, 4, THREADS, MODE_FRONTIER>(p, p.top, ta, bq / NW + (w < bq % NW ? 1u : 0u));
                run_phase<PRF, 4, THREADS, MODE_FRONTIER>(p, p.top, ta);
            }
            if (stamp) stamp[2] = global_ns();
            grid_barrier(p.grid_bar, p.grid_bar_target);
            if (stamp) stamp[3] = global_ns();
            if (blockIdx.x == 0)   /* nobody draws top-phase tickets any more: re-arm them for the next launch */
                for (uint32_t i = tid; i < p.rearm_words; i += THREADS) p.rearm[i] = 0u;
        }
    }
    if constexpr (mode_traits(MODE).units) run_units<PRF, NV, THREADS, MODE>(p, p.main, ta);
    else run_phase<PRF, NV, THREADS, MODE>(p, p.main, ta);
    if (stamp) stamp[4] = global_ns();
}

/* MAC-only pass for wide entries: leaves come from the cache written by the first fused
 * pass, rows are broadcast loads as in the fused kernel.  One warp = 32 keys x one range
 * of leaf positions; pure streaming (HBM/L2 -> IMAD), no PRF work. */
template <int NV>
__global__ void __launch_bounds__(256, 2) dpf_mac_kernel(const __grid_constant__ MacParams p)
{
    const int lane = threadIdx.x & 31;
    const uint64_t warp_global = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint64_t warps_total = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t items = (uint64_t)p.key_groups * p.ranges_per_group;
    const uint64_t len = (p.n_local + p.ranges_per_group - 1) / p.ranges_per_group;
    for (uint64_t w = warp_global; w < items; w += warps_total) {
        /* range is the fast index (key-group-fast ordering measured slower: 30.4 vs 29.2 ms at E=128) */
        const uint32_t kg = (uint32_t)(w / p.ranges_per_group);
        const uint32_t r = (uint32_t)(w - (uint64_t)kg * p.ranges_per_group);
        const uint64_t begin = (uint64_t)r * len;
        const uint64_t end = begin + len < p.n_local ? begin + len : p.n_local;
        uint32_t acc[4 * NV];
#pragma unroll
        for (int e = 0; e < 4 * NV; e++) acc[e] = 0;
        const uint32_t *leaf = p.leaf_cache + ((size_t)kg * p.n_local + begin) * 32 + lane;
        const uint4 *row = p.table + begin * p.row_stride_v + p.col_off_v;
        uint64_t pos = begin;
        for (; pos + 4 <= end; pos += 4) {   /* 4 leaves per trip: 4 independent load streams in flight */
            uint32_t v[4];
#pragma unroll
            for (int u = 0; u < 4; u++) v[u] = __ldg(leaf + 32 * u);
#pragma unroll
            for (int j = 0; j < NV; j++) {
                uint4 t[4];
#pragma unroll
                for (int u = 0; u < 4; u++) t[u] = __ldg(row + (size_t)u * p.row_stride_v + j);
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    acc[4 * j + 0] += v[u] * t[u].x;
                    acc[4 * j + 1] += v[u] * t[u].y;
                    acc[4 * j + 2] += v[u] * t[u].z;
                    acc[4 * j + 3] += v[u] * t[u].w;
                }
            }
            leaf += 128;
            row += (size_t)4 * p.row_stride_v;
        }
        for (; pos < end; pos++) {
            const uint32_t v = __ldg(leaf);
#pragma unroll
            for (int j = 0; j < NV; j++) {
                const uint4 t = __ldg(row + j);
                acc[4 * j + 0] += v * t.x;
                acc[4 * j + 1] += v * t.y;
                acc[4 * j + 2] += v * t.z;
                acc[4 * j + 3] += v * t.w;
            }
            leaf += 32;
            row += p.row_stride_v;
        }
        const int key = (int)kg * 32 + lane;
        if (key < p.nkeys) {
            uint32_t *o = p.out + (size_t)key * p.out_stride + p.col_off;
#pragma unroll
            for (int e = 0; e < 4 * NV; e++)
                if ((uint32_t)e >= p.col_skip && (uint32_t)e < p.ncols) atomicAdd(o + e, acc[e]);
        }
    }
}

/* ---- TMA-staged MAC pass ---------------------------------------------------------------------
 * Same arithmetic as dpf_mac_kernel, organised as a producer/consumer pipeline: one warp issues
 * cp.async.bulk copies (table-row slices and cached leaves, global -> shared, completion counted
 * on an mbarrier), eight consumer warps -- one key group each, all on the SAME leaf positions,
 * so a row slice staged once is multiplied against 8 x 32 keys -- do LDS + IMAD only.  The
 * register-staged variant above is latency bound (16 dependent load phases per trip); this one
 * is bound by the FMA pipe. */

template <int NV>
struct MacTmaShape {
    enum { P = 32, STAGES = 3, GROUPS = 8, ROW_BYTES = NV * 16, LEAF_TILE = P * 128,
           STAGE_BYTES = GROUPS * LEAF_TILE + P * ROW_BYTES, SMEM = STAGES * STAGE_BYTES + 64,
           THREADS = (GROUPS + 1) * 32 };
};

template <int NV>
__global__ void __launch_bounds__(MacTmaShape<NV>::THREADS, 1) dpf_mac_tma_kernel(const __grid_constant__ MacParams p)
{
    typedef MacTmaShape<NV> S;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t smem0 = (uint32_t)__cvta_generic_to_shared(g_dyn_smem);
    const uint32_t bars = smem0 + S::STAGES * S::STAGE_BYTES;   /* full[STAGES], empty[STAGES] */
    if (threadIdx.x == 0) {
        for (int i = 0; i < S::STAGES; i++) {
            tma::mbar_init(bars + 8 * i, 1);                       /* producer's expect_tx arrival */
            tma::mbar_init(bars + 8 * (S::STAGES + i), S::GROUPS); /* one arrival per consumer warp */
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const uint32_t kg_blocks = ((uint32_t)p.key_groups + S::GROUPS - 1) / S::GROUPS;
    const uint64_t items = (uint64_t)kg_blocks * p.ranges_per_group;
    const uint64_t len = (p.n_local + p.ranges_per_group - 1) / p.ranges_per_group;
    uint32_t seq = 0;   /* tiles issued / consumed so far: stage = seq % STAGES, phase = (seq / STAGES) & 1 */

    for (uint64_t it = blockIdx.x; it < items; it += gridDim.x) {
        const uint32_t kgb = (uint32_t)(it / p.ranges_per_group);
        const uint32_t r = (uint32_t)(it - (uint64_t)kgb * p.ranges_per_group);
        const uint64_t begin = (uint64_t)r * len;
        const uint64_t end = begin + len < p.n_local ? begin + len : p.n_local;
        const uint32_t kg0 = kgb * S::GROUPS;
        const uint32_t ngroups = min((uint32_t)S::GROUPS, (uint32_t)p.key_groups - kg0);

        if (warp == S::GROUPS) {
            /* ===== producer warp ===== */
            for (uint64_t pos = begin; pos < end; pos += S::P, seq++) {
                const uint32_t stage = seq % S::STAGES, phase = (seq / S::STAGES) & 1u;
                const uint32_t cnt = (uint32_t)min((uint64_t)S::P, end - pos);
                const uint32_t sbase = smem0 + stage * S::STAGE_BYTES;
                const uint32_t full = bars + 8 * stage, empty = bars + 8 * (S::STAGES + stage);
                tma::mbar_wait(empty, phase ^ 1u);     /* consumers have released this stage */
                if (lane == 0) tma::mbar_expect_tx(full, cnt * (128u * ngroups + S::ROW_BYTES));
                __syncwarp();
                if ((uint32_t)lane < ngroups)          /* cached leaves: one contiguous slab per key group */
                    tma::bulk_g2s(sbase + lane * S::LEAF_TILE,
                                  p.leaf_cache + ((size_t)(kg0 + lane) * p.n_local + pos) * 32, cnt * 128u, full);
                for (uint32_t i = lane; i < cnt; i += 32)   /* one row slice per leaf position */
                    tma::bulk_g2s(sbase + S::GROUPS * S::LEAF_TILE + i * S::ROW_BYTES,
                                  p.table + (pos + i) * p.row_stride_v + p.col_off_v, S::ROW_BYTES, full);
            }
        } else {
            /* ===== consumer warps: warp w = key group kg0 + w ===== */
            const bool active = (uint32_t)warp < ngroups;
            uint32_t acc[4 * NV];
#pragma unroll
            for (int e = 0; e < 4 * NV; e++) acc[e] = 0;
            for (uint64_t pos = begin; pos < end; pos += S::P, seq++) {
                const uint32_t stage = seq % S::STAGES, phase = (seq / S::STAGES) & 1u;
                const uint32_t cnt = (uint32_t)min((uint64_t)S::P, end - pos);
                const unsigned char *sbase = g_dyn_smem + stage * S::STAGE_BYTES;
                tma::mbar_wait(bars + 8 * stage, phase);   /* the bytes have landed */
                if (active) {
                    const uint32_t *leaf = reinterpret_cast<const uint32_t *>(sbase + warp * S::LEAF_TILE) + lane;
                    const uint4 *rows = reinterpret_cast<const uint4 *>(sbase + S::GROUPS * S::LEAF_TILE);
#pragma unroll 2
                    for (uint32_t i = 0; i < cnt; i++) {
                        const uint32_t v = leaf[i * 32];
#pragma unroll
                        for (int j = 0; j < NV; j++) {
                            const uint4 t = rows[i * NV + j];
                            acc[4 * j + 0] += v * t.x;
                            acc[4 * j + 1] += v * t.y;
                            acc[4 * j + 2] += v * t.z;
                            acc[4 * j + 3] += v * t.w;
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) tma::mbar_arrive(bars + 8 * (S::STAGES + stage));
            }
            const int key = (int)(kg0 + warp) * 32 + lane;
            if (active && key < p.nkeys) {
                uint32_t *o = p.out + (size_t)key * p.out_stride + p.col_off;
#pragma unroll
                for (int e = 0; e < 4 * NV; e++)
                    if ((uint32_t)e >= p.col_skip && (uint32_t)e < p.ncols) atomicAdd(o + e, acc[e]);
            }
        }
    }
}

__global__ void __launch_bounds__(256) sum_partials_kernel(uint32_t *__restrict__ dst, const PeerParts parts, size_t words)
{
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)gridDim.x * blockDim.x;
    if ((words & 3u) == 0) {   /* results are [B][E] int32 from cudaMalloc: 16-byte aligned whenever the count allows */
        uint4 *d4 = reinterpret_cast<uint4 *>(dst);
        for (size_t i = tid; i < words / 4; i += nthr) {
            uint4 a = d4[i];
            for (int k = 0; k < parts.n; k++) {
                const uint4 b = __ldcg(reinterpret_cast<const uint4 *>(parts.p[k]) + i);   /* peer memory over NVLink */
                a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
            }
            d4[i] = a;
        }
    } else {
        for (size_t i = tid; i < words; i += nthr) {
            uint32_t a = dst[i];
            for (int k = 0; k < parts.n; k++) a += __ldcg(parts.p[k] + i);
            dst[i] = a;
        }
    }
}

__global__ void probe_smem_kernel(uint32_t *out)
{
    if (threadIdx.x == 0) *out = (uint32_t)__cvta_generic_to_shared(g_dyn_smem);
}

/* table[P.device_row(r)][c] = chunk[q][c] for q < count, c < cols, where r is the natural row of own row j = first + q:
 * own leaf j >> lane_bits is natural leaf ((j >> lane_bits) << shift) | own_val. */
__global__ void fill_table_kernel(const int32_t *__restrict__ chunk, uint64_t first, uint64_t count, int32_t *__restrict__ table,
                                  const RowPlacement P, int cols, int stride)
{
    const uint64_t total = count * (uint64_t)cols;
    const uint64_t lane_mask = (1u << P.lane_bits) - 1u;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t q = i / (uint64_t)cols;
        const int c = (int)(i - q * (uint64_t)cols);
        const uint64_t j = first + q;
        const uint64_t r = ((((j >> P.lane_bits) << P.shift) | P.own_val) << P.lane_bits) | (j & lane_mask);
        table[P.device_row((int64_t)r) * (uint64_t)stride + c] = chunk[i];
    }
}

/* row update, step 1: natural row -> device row (UpdateParams) or the skip marker, occurrence number j */
__global__ void __launch_bounds__(256) update_map_kernel(const UpdateParams u, uint32_t *__restrict__ pos,
                                                         uint32_t *__restrict__ ord)
{
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < u.count; j += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = u.idx[j];
        RowPlacement P = u.place;
        bool in_range = true;
        if (u.bins) {
            const int32_t g = u.bins[j];
            in_range = g >= 0 && g < u.nbins;
            if (in_range) P = u.bin_place[g];
        }
        pos[j] = in_range && P.owns(i) ? (uint32_t)P.device_row(i) : u.table_rows;
        ord[j] = (uint32_t)j;
    }
}

/* row update, step 3: positions sorted stably, so the last occurrence of a position ends its run;
 * one warp copies that occurrence's row, 16 bytes per lane and step when the rows allow it.  (Scalar
 * arguments: reading them out of the UpdateParams struct costs this loop a spill.) */
__global__ void __launch_bounds__(256) update_scatter_kernel(const int32_t *__restrict__ rows, int32_t *__restrict__ table,
                                                             const uint32_t *__restrict__ pos, const uint32_t *__restrict__ ord,
                                                             int64_t count, uint32_t skip, int cols, int stride, int vec4)
{
    const int lane = (int)(threadIdx.x & 31u);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x / 32);
    for (int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; k < count; k += nwarps) {
        const uint32_t p = pos[k];
        if (p == skip) break;                               /* skipped entries sort last */
        if (k + 1 < count && pos[k + 1] == p) continue;     /* a later occurrence wins  */
        const int32_t *src = rows + (size_t)ord[k] * (size_t)cols;
        int32_t *dst = table + (size_t)p * (size_t)stride;
        if (vec4) {
            const int4 *s4 = reinterpret_cast<const int4 *>(src);
            int4 *d4 = reinterpret_cast<int4 *>(dst);
            for (int c = lane; c < cols / 4; c += 32) d4[c] = s4[c];
        } else {
            for (int c = lane; c < cols; c += 32) dst[c] = src[c];
        }
    }
}

/* An instantiated evaluation kernel: its entry point, and whether its attributes are set on each device
 * (1 = set, 0 = never).  Function attributes belong to the (kernel, device) pair for the whole process, not
 * to one context, so the dynamic shared-memory ceiling is set once, to the most the kernel can take
 * (eval_max_smem), and every launch passes its own size below it.  Contexts on different host threads may
 * race to set it; they all write the same values, so a duplicate set is harmless. */
struct EvalKernel {
    const void *fn;
    std::atomic<int> *configured;   /* [64] */
};

template <int PRF, int NV, int MODE>
EvalKernel eval_kernel()
{
    static std::atomic<int> configured[64];
    return EvalKernel{reinterpret_cast<const void *>(dpf_eval_kernel<PRF, NV, MODE>), configured};
}

/* The instantiated kernels of one PRF.  Every mode runs at 16 columns per pass (nv = 4); the fused
 * modes of standard and early-terminated keys also at 32, the standard one at 64 as well.  Grouped
 * evaluation (every kind of key) and XOR-shared keys take 16 columns per pass, and the modes that never
 * touch the table need no other width. */
template <int PRF>
EvalKernel eval_kernel_of(int nv, int mode)
{
    if (nv == 4) {
        switch (mode) {
        case MODE_FUSED: return eval_kernel<PRF, 4, MODE_FUSED>();
        case MODE_EXPAND: return eval_kernel<PRF, 4, MODE_EXPAND>();
        case MODE_FRONTIER: return eval_kernel<PRF, 4, MODE_FRONTIER>();
        case MODE_GROUPED: return eval_kernel<PRF, 4, MODE_GROUPED>();
        case MODE_FUSED_ET: return eval_kernel<PRF, 4, MODE_FUSED_ET>();
        case MODE_EXPAND_ET: return eval_kernel<PRF, 4, MODE_EXPAND_ET>();
        case MODE_GROUPED_ET: return eval_kernel<PRF, 4, MODE_GROUPED_ET>();
        case MODE_FUSED_XOR: return eval_kernel<PRF, 4, MODE_FUSED_XOR>();
        case MODE_EXPAND_XOR: return eval_kernel<PRF, 4, MODE_EXPAND_XOR>();
        case MODE_GROUPED_XOR: return eval_kernel<PRF, 4, MODE_GROUPED_XOR>();
        case MODE_GROUPED_DEV: return eval_kernel<PRF, 4, MODE_GROUPED_DEV>();
        case MODE_GROUPED_ET_DEV: return eval_kernel<PRF, 4, MODE_GROUPED_ET_DEV>();
        case MODE_GROUPED_XOR_DEV: return eval_kernel<PRF, 4, MODE_GROUPED_XOR_DEV>();
        case MODE_FUSED_TMA:       /* AES: no shared memory left beside the tables */
            if constexpr (PRF != PRF_AES128) return eval_kernel<PRF, 4, MODE_FUSED_TMA>();
            break;
        case MODE_FUSED_COLSPLIT:   /* Salsa/ChaCha bind the ALU pipe, not the data pipe */
            if constexpr (PRF == PRF_AES128) return eval_kernel<PRF, 4, MODE_FUSED_COLSPLIT>();
            break;
        }
    } else if (nv == 8) {
        if (mode == MODE_FUSED) return eval_kernel<PRF, 8, MODE_FUSED>();
        if (mode == MODE_FUSED_ET) return eval_kernel<PRF, 8, MODE_FUSED_ET>();
    } else if (nv == 16) {
        if (mode == MODE_FUSED) return eval_kernel<PRF, 16, MODE_FUSED>();
    }
    return EvalKernel{nullptr, nullptr};
}

/* (prf, nv, mode) -> its kernel, or {nullptr} when it is not instantiated */
EvalKernel find_eval_kernel(int prf, int nv, int mode)
{
    switch (prf) {
    case PRF_DUMMY: return eval_kernel_of<PRF_DUMMY>(nv, mode);
    case PRF_SALSA20: return eval_kernel_of<PRF_SALSA20>(nv, mode);
    case PRF_CHACHA20: return eval_kernel_of<PRF_CHACHA20>(nv, mode);
    case PRF_AES128: return eval_kernel_of<PRF_AES128>(nv, mode);
    default: return EvalKernel{nullptr, nullptr};
    }
}

/* The most dynamic shared memory one block of kernel `fn` may take on the current device: the opt-in limit
 * less the kernel's static shared memory */
cudaError_t kernel_max_smem(const void *fn, int *bytes)
{
    cudaFuncAttributes a;
    cudaError_t e = cudaFuncGetAttributes(&a, fn);
    if (e != cudaSuccess) return e;
    int dev = 0, optin = 0;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
    if ((e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)) != cudaSuccess) return e;
    *bytes = optin - (int)a.sharedSizeBytes;
    return cudaSuccess;
}

}  // namespace

cudaError_t probe_dynamic_smem_base(uint32_t *base, cudaStream_t stream)
{
    uint32_t *d = nullptr;
    cudaError_t e = cudaMalloc(&d, sizeof(uint32_t));
    if (e != cudaSuccess) return e;
    probe_smem_kernel<<<1, 32, 16, stream>>>(d);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(base, d, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    cudaFree(d);
    return e;
}

cudaError_t upload_aes_table(const uint32_t *te0_256)
{
    return cudaMemcpyToSymbol(c_te0, te0_256, 256 * sizeof(uint32_t));
}

cudaError_t launch_eval(int prf, int nv, int mode, const EvalParams &p, int grid, size_t smem, cudaStream_t stream)
{
    const EvalKernel k = find_eval_kernel(prf, nv, mode);
    if (k.fn == nullptr) return cudaErrorInvalidValue;
    /* the column split trades leaf values across the four lanes of a key quad, which must be four keys */
    if (mode_traits(mode).row_load == ROWS_COLSPLIT && p.kpw_log2 < 2) return cudaErrorInvalidValue;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64 || !k.configured[dev].load(std::memory_order_acquire)) {
        /* the ceiling, not this launch's size: a smaller value set by another thread between its check and its
         * launch would make that launch fail */
        int max_smem = 0;
        if ((e = kernel_max_smem(k.fn, &max_smem)) != cudaSuccess) return e;
        e = cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
        if (e != cudaSuccess) return e;
        /* the kernels live in shared memory; L1 only sees broadcast table rows */
        e = cudaFuncSetAttribute(k.fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 64) k.configured[dev].store(1, std::memory_order_release);
    }
    const dim3 block((unsigned)eval_block_shape(prf, nv, mode).threads);
    void *args[] = {const_cast<EvalParams *>(&p)};
    if (p.fuse_top) return cudaLaunchCooperativeKernel(k.fn, dim3((unsigned)grid), block, args, smem, stream);
    cudaLaunchKernel(k.fn, dim3((unsigned)grid), block, args, smem, stream);   /* as <<<>>>: read back below */
    return cudaGetLastError();
}

cudaError_t eval_max_smem(int prf, int nv, int mode, int *bytes)
{
    const EvalKernel k = find_eval_kernel(prf, nv, mode);
    if (k.fn == nullptr) return cudaErrorInvalidValue;
    return kernel_max_smem(k.fn, bytes);
}

cudaError_t launch_mac_tma(const MacParams &p, int grid, cudaStream_t stream)
{
    typedef MacTmaShape<16> S;
    auto kern = dpf_mac_tma_kernel<16>;
    /* every launch takes the same S::SMEM, so every thread that sets the attribute writes the same value */
    static std::atomic<int> configured[64];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64 || !configured[dev].load(std::memory_order_acquire)) {
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S::SMEM);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 64) configured[dev].store(1, std::memory_order_release);
    }
    kern<<<grid, (int)S::THREADS, (int)S::SMEM, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_mac(int nv, const MacParams &p, int grid, cudaStream_t stream)
{
    if (nv == 4) dpf_mac_kernel<4><<<grid, 256, 0, stream>>>(p);
    else if (nv == 8) dpf_mac_kernel<8><<<grid, 256, 0, stream>>>(p);
    else if (nv == 16) dpf_mac_kernel<16><<<grid, 256, 0, stream>>>(p);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

cudaError_t launch_sum_partials(uint32_t *dst, const PeerParts &parts, size_t words, int sm_count, cudaStream_t stream)
{
    if (parts.n <= 0 || words == 0) return cudaSuccess;
    int grid = (int)std::min<size_t>((words / 4 + 255) / 256 + 1, (size_t)std::max(sm_count, 1) * 4);
    sum_partials_kernel<<<grid, 256, 0, stream>>>(dst, parts, words);
    return cudaGetLastError();
}

cudaError_t launch_fill_table(const int32_t *chunk, uint64_t first, uint64_t count, int32_t *table, const RowPlacement &P,
                              int cols, int stride, int sm_count, cudaStream_t stream)
{
    const uint64_t total = count * (uint64_t)cols;
    const uint64_t cap = (uint64_t)std::max(sm_count, 1) * 16;
    int grid = (int)std::min<uint64_t>((total + 255) / 256, cap);
    if (grid < 1) grid = 1;
    fill_table_kernel<<<grid, 256, 0, stream>>>(chunk, first, count, table, P, cols, stride);
    return cudaGetLastError();
}

cudaError_t update_temp_bytes(int64_t count, int end_bit, size_t *bytes)
{
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                           (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)count, 0, end_bit);
}

cudaError_t launch_update_rows(const UpdateParams &u, const UpdateWork &w, int end_bit, int sm_count, cudaStream_t stream)
{
    if (u.count <= 0) return cudaSuccess;
    const int64_t cap = (int64_t)std::max(sm_count, 1) * 16;
    const int grid_map = (int)std::max<int64_t>(1, std::min<int64_t>((u.count + 255) / 256, cap));
    update_map_kernel<<<grid_map, 256, 0, stream>>>(u, w.pos_in, w.ord_in);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    size_t temp_bytes = w.temp_bytes;
    e = cub::DeviceRadixSort::SortPairs(w.temp, temp_bytes, w.pos_in, w.pos_out, w.ord_in, w.ord_out, (int)u.count, 0,
                                        end_bit, stream);
    if (e != cudaSuccess) return e;
    const bool vec4 = (u.cols & 3) == 0 && (reinterpret_cast<uintptr_t>(u.rows) & 15u) == 0;
    const int grid_scatter = (int)std::max<int64_t>(1, std::min<int64_t>((u.count + 7) / 8, cap));
    update_scatter_kernel<<<grid_scatter, 256, 0, stream>>>(u.rows, u.table, w.pos_out, w.ord_out, u.count, u.table_rows,
                                                            u.cols, u.stride, vec4 ? 1 : 0);
    return cudaGetLastError();
}

}  // namespace b200dpf
