// Microbenchmark: integer-pipe issue rates on one SM, so the integer roofline of the DPF kernels
// rests on measured numbers (SURVEY.md section 7.4; VERDICT r1 item 5).
//
// For each instruction class the kernel runs CH independent dependency chains per thread with
// 16 warps per SM (4 per scheduler) and reports warp-instructions per clock per SM, from the
// SM's own cycle counter (clock64), so the number does not depend on the clock the board runs at.
//   alu pipe : LOP3, SHF (funnel shift), PRMT, IADD3
//   fma pipe : IMAD (mad.lo), IMAD.WIDE (mul.wide), IMAD.HI (mul.hi)
//   lsu      : conflict-free 32-bit shared-memory loads (the AES T-table access pattern)
//   mixes    : LOP3+IMAD, LOP3+SHF+IMAD (can the two pipes issue in the same clock?), LDS+PRMT+LOP3
//   lsu + ldg: the LDS steps plus 3 warp-uniform (broadcast) LDG.128 per 128 LDS, the ratio of the
//              fused AES kernel's table-row loads (8 per leaf pair of ~300 lookups); each load hits
//              one 64-byte row of a 4 MiB buffer (L2-resident), consumed by IMADs like the MAC.  That
//              ratio holds inside a leaf pair only; per AES height-2 unit (4 leaves: 1,268 lookups, 4
//              rows) it is 16 per 1,268, the "16 per 1280 LDS" line
//   tensor-core inner product: the LDS steps plus, per 1280 LDS, what an 8-key x 4-subtree lane
//              mapping with the inner product on IMMA would issue per unit: 4 LDG.64 (no broadcast),
//              24 PRMT and 10 IMMA.16816.U8.U8; and the same without the IMMA as a control
//   quarter rounds: Salsa20 / ChaCha as the kernels write them, and variants that move some of
//   the rotates to the fma pipe as IMAD.WIDE (x*2^r = {x<<r, x>>(32-r)}; the halves are disjoint,
//   so  b ^ rotl(t,r) == lop3.xor(b, lo, hi)).
// Which SASS instruction each PTX line became can be checked with cuobjdump -sass.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o bin/int_pipes int_pipes.cu
// Output: one JSON object per line on stdout.
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#define CH 8          // independent chains per thread
#define UNROLL 16     // ops per chain per loop trip

enum Op { OP_LOP3, OP_SHF, OP_PRMT, OP_IADD3, OP_IMAD, OP_IMADWIDE, OP_IMADHI, OP_LDS,
          OP_MIX_LOP3_IMAD, OP_MIX_LOP3_SHF_IMAD, OP_MIX_LDS_PRMT_LOP3, OP_MIX_LOP3_IMADWIDE, OP_LDS_LDG,
          OP_LDS_LDG_UNIT, OP_LDS_MMA_UNIT, OP_LDS_LDG64_UNIT };

template <int OP>
__device__ __forceinline__ void step(uint32_t &x, uint32_t y, uint32_t z, uint32_t smem_lane)
{
    if (OP == OP_LOP3) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x) : "r"(y), "r"(z));
    } else if (OP == OP_SHF) {
        asm volatile("shf.l.wrap.b32 %0, %0, %0, 7;" : "+r"(x));
    } else if (OP == OP_PRMT) {
        asm volatile("prmt.b32 %0, %0, %1, 0x2103;" : "+r"(x) : "r"(y));
    } else if (OP == OP_IADD3) {
        /* three-input add: ptxas emits IADD3 (alu pipe) */
        asm volatile("{\n\t.reg .u32 t;\n\tadd.u32 t, %0, %1;\n\tadd.u32 %0, t, %2;\n\t}" : "+r"(x) : "r"(y), "r"(z));
    } else if (OP == OP_IMAD) {
        asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(x) : "r"(y), "r"(z));
    } else if (OP == OP_IMADWIDE) {
        asm volatile("{\n\t.reg .u64 t;\n\t.reg .u32 lo, hi;\n\tmul.wide.u32 t, %0, 128;\n\tmov.b64 {lo, hi}, t;\n\t"
                     "lop3.b32 %0, lo, hi, %1, 0x96;\n\t}" : "+r"(x) : "r"(y));
    } else if (OP == OP_IMADHI) {
        asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(x) : "r"(y));
    } else if (OP == OP_LDS || OP == OP_LDS_LDG || OP == OP_LDS_LDG_UNIT || OP == OP_LDS_MMA_UNIT || OP == OP_LDS_LDG64_UNIT) {
        uint32_t a;
        asm volatile("prmt.b32 %0, %1, %2, 0x7604;" : "=r"(a) : "r"(x), "r"(smem_lane));
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(x) : "r"(a));
    } else if (OP == OP_MIX_LOP3_IMAD) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x) : "r"(y), "r"(z));
        asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(x) : "r"(y), "r"(z));
    } else if (OP == OP_MIX_LOP3_SHF_IMAD) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x) : "r"(y), "r"(z));
        asm volatile("shf.l.wrap.b32 %0, %0, %0, 7;" : "+r"(x));
        asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(x) : "r"(y), "r"(z));
    } else if (OP == OP_MIX_LDS_PRMT_LOP3) {
        uint32_t a, v;
        asm volatile("prmt.b32 %0, %1, %2, 0x7604;" : "=r"(a) : "r"(x), "r"(smem_lane));
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x) : "r"(v), "r"(z));
    } else if (OP == OP_MIX_LOP3_IMADWIDE) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x) : "r"(y), "r"(z));
        asm volatile("{\n\t.reg .u64 t;\n\t.reg .u32 lo, hi;\n\tmul.wide.u32 t, %0, 128;\n\tmov.b64 {lo, hi}, t;\n\t"
                     "lop3.b32 %0, lo, hi, %1, 0x96;\n\t}" : "+r"(x) : "r"(y));
    }
}

/* instructions one step<OP> issues (for the rate): {alu, fma, lsu} */
struct Mix { int alu, fma, lsu; };
__host__ __device__ constexpr Mix mix_of(int op)
{
    return op == OP_LOP3 || op == OP_SHF || op == OP_PRMT || op == OP_IADD3 ? Mix{1, 0, 0}
         : op == OP_IMAD || op == OP_IMADHI ? Mix{0, 1, 0}
         : op == OP_IMADWIDE ? Mix{1, 1, 0}
         : op == OP_LDS || op == OP_LDS_LDG || op == OP_LDS_LDG_UNIT || op == OP_LDS_MMA_UNIT || op == OP_LDS_LDG64_UNIT ? Mix{1, 0, 1}
         : op == OP_MIX_LOP3_IMAD ? Mix{1, 1, 0}
         : op == OP_MIX_LOP3_SHF_IMAD ? Mix{2, 1, 0}
         : op == OP_MIX_LDS_PRMT_LOP3 ? Mix{2, 0, 1}
         : Mix{2, 1, 0};
}

// 256 entries x 256 bytes (32 lanes x 4 bytes used), placed at a 64 KiB-aligned shared-window
// address like the AES kernel's tables, so one PRMT (index byte -> byte 1 of base+4*lane) is the address
extern __shared__ __align__(16) unsigned char s_raw[];
#define TAB_SMEM (128 * 1024 + 16)

template <int OP>
#define ROWS_MASK 65535u   /* 64 KiB rows of 64 bytes = 4 MiB */
__global__ void __launch_bounds__(512, 1) pipe_kernel(uint32_t *out, long long *cycles, int iters, const uint4 *rows)
{
    const uint32_t base = (uint32_t)__cvta_generic_to_shared(s_raw);
    const uint32_t tab = (base + 65535u) & ~65535u;            /* 64 KiB-aligned window address inside the 128 KiB */
    unsigned char *tabp = s_raw + (tab - base);
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x)
        *reinterpret_cast<uint32_t *>(tabp + (i >> 5) * 256 + (i & 31) * 4) = i * 2654435761u;
    __syncthreads();
    const uint32_t smem_lane = tab + (threadIdx.x & 31) * 4;
    uint32_t x[CH];
#pragma unroll
    for (int c = 0; c < CH; c++) x[c] = threadIdx.x * 2654435761u + c * 40503u + blockIdx.x;
    const uint32_t y = x[0] | 1u, z = x[1] ^ 0x5bd1e995u;
    const uint32_t warp_id = blockIdx.x * 16u + (threadIdx.x >> 5);
    uint32_t sink = 0;
    uint32_t d0 = 0, d1 = 0, d2 = 0, d3 = 0, a0 = y, a1 = z, bp = 0;
    uint2 ga = make_uint2(0, 0), gb = make_uint2(0, 0);
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        /* the *_UNIT mixes repeat every 5 trips = 640 LDS, half of an AES height-2 unit's 1,268 lookups */
        const int ph = it % 5;
        const uint32_t row = ((uint32_t)it * 2654435761u + warp_id) & ROWS_MASK;
#pragma unroll
        for (int u = 0; u < UNROLL; u++) {
#pragma unroll
            for (int c = 0; c < CH; c++) step<OP>(x[c], y, z, smem_lane);
            if (OP == OP_LDS_LDG && u % 5 == 2) {   /* u = 2, 7, 12: words 0..2 of this trip's row */
                const uint4 r = __ldg(rows + (size_t)row * 4 + u / 5);
                sink += r.x * y + r.y * z + r.z * y + r.w * z;
            }
            /* the fused kernel's row loads: 16 broadcast LDG.128 (4 rows x 64 bytes) per unit = 8 per 5 trips */
            if (OP == OP_LDS_LDG_UNIT && (u == 2 || (u == 9 && ph < 3))) {
                const uint4 r = __ldg(rows + (size_t)row * 4 + (u == 2 ? 0 : 1));
                sink += r.x * y + r.y * z + r.z * y + r.w * z;
            }
            /* inner product on the tensor cores (8 keys x 4 subtrees per warp): per unit 4 LDG.64 (lane L:
             * row of subtree slot L & 3, columns 2 (L >> 2) and +1), 24 PRMT byte-plane splits and 10
             * IMMA.16816.U8.U8 = per 5 trips 2 / 12 / 5.  LDG64_UNIT: the same without the IMMA (its
             * operands are folded into the sink instead) */
            if (OP == OP_LDS_MMA_UNIT || OP == OP_LDS_LDG64_UNIT) {
                if (u == 2 && ph == 0) {
                    const uint2 *r = reinterpret_cast<const uint2 *>(rows) + ((threadIdx.x >> 2) & 7);
                    ga = __ldg(r + (size_t)((row + (threadIdx.x & 3)) & ROWS_MASK) * 8);
                    gb = __ldg(r + (size_t)((row + 4 + (threadIdx.x & 3)) & ROWS_MASK) * 8);
                }
                if (u == 5) {
                    bp = __byte_perm(x[0], x[1], 0x5140);
                    bp = __byte_perm(bp, x[2], 0x5410);
                }
                if (u == 11 && ph == 0) {
                    a0 = __byte_perm(ga.x, gb.x, 0x5140);
                    a1 = __byte_perm(ga.y, gb.y, 0x7362);
                }
                if (u == 13 && OP == OP_LDS_LDG64_UNIT) sink ^= a0 ^ a1 ^ bp;
                if (u == 13 && OP == OP_LDS_MMA_UNIT)
                    asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                                 : "+r"(d0), "+r"(d1), "+r"(d2), "+r"(d3) : "r"(a0), "r"(a1), "r"(bp));
            }
        }
    }
    __syncthreads();
    const long long t1 = clock64();
    uint32_t acc = sink ^ d0 ^ d1 ^ d2 ^ d3;
#pragma unroll
    for (int c = 0; c < CH; c++) acc ^= x[c];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

/* ---- quarter-round variants ---------------------------------------------------------------- */
__device__ __forceinline__ uint32_t rotl_shf(uint32_t v, int r) { return __funnelshift_l(v, v, r); }

template <int R>
__device__ __forceinline__ void wide_rot(uint32_t v, uint32_t &lo, uint32_t &hi)
{
    asm("{\n\t.reg .u64 t;\n\tmul.wide.u32 t, %2, %3;\n\tmov.b64 {%0, %1}, t;\n\t}" : "=r"(lo), "=r"(hi) : "r"(v), "n"(1u << R));
}
__device__ __forceinline__ uint32_t xor3(uint32_t a, uint32_t b, uint32_t c)
{
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
/* b ^= rotl(t, R): MASKBIT ? fma-pipe form : alu-pipe form */
template <bool FMA, int R>
__device__ __forceinline__ uint32_t xor_rot(uint32_t b, uint32_t t)
{
    if (FMA) {
        uint32_t lo, hi;
        wide_rot<R>(t, lo, hi);
        return xor3(b, lo, hi);
    }
    return b ^ rotl_shf(t, R);
}

template <int MASK>
__device__ __forceinline__ void salsa_qr(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t &d)
{
    b = xor_rot<(MASK & 1) != 0, 7>(b, a + d);
    c = xor_rot<(MASK & 2) != 0, 9>(c, b + a);
    d = xor_rot<(MASK & 4) != 0, 13>(d, c + b);
    a = xor_rot<(MASK & 8) != 0, 18>(a, d + c);
}

/* d = rotl(d ^ a, R) with the rotate on the fma pipe: the rotated word is rebuilt with one add */
template <bool FMA, int R>
__device__ __forceinline__ uint32_t rot_xor(uint32_t d, uint32_t a)
{
    if (FMA) {
        uint32_t lo, hi;
        wide_rot<R>(d ^ a, lo, hi);
        return lo + hi;
    }
    return rotl_shf(d ^ a, R);
}

template <int MASK>
__device__ __forceinline__ void chacha_qr(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t &d)
{
    a += b; d = rot_xor<(MASK & 1) != 0, 16>(d, a);
    c += d; b = rot_xor<(MASK & 2) != 0, 12>(b, c);
    a += b; d = rot_xor<(MASK & 4) != 0, 8>(d, a);
    c += d; b = rot_xor<(MASK & 8) != 0, 7>(b, c);
}

template <int KIND, int MASK>   /* KIND 0 salsa, 1 chacha */
__global__ void __launch_bounds__(512, 1) qr_kernel(uint32_t *out, long long *cycles, int iters)
{
    uint32_t s[4][4];
#pragma unroll
    for (int q = 0; q < 4; q++)
#pragma unroll
        for (int w = 0; w < 4; w++) s[q][w] = threadIdx.x * 2654435761u + (q * 4 + w) * 40503u + blockIdx.x;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
#pragma unroll
            for (int q = 0; q < 4; q++) {
                if (KIND == 0) salsa_qr<MASK>(s[q][0], s[q][1], s[q][2], s[q][3]);
                else chacha_qr<MASK>(s[q][0], s[q][1], s[q][2], s[q][3]);
            }
            /* rotate the roles of the words like the column/diagonal rounds do */
#pragma unroll
            for (int q = 0; q < 4; q++) { const uint32_t t = s[q][1]; s[q][1] = s[(q + 1) & 3][1]; s[(q + 1) & 3][1] = t; }
        }
    }
    __syncthreads();
    const long long t1 = clock64();
    uint32_t acc = 0;
#pragma unroll
    for (int q = 0; q < 4; q++)
#pragma unroll
        for (int w = 0; w < 4; w++) acc ^= s[q][w];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

static uint32_t *g_out;
static long long *g_cycles;
static uint4 *g_rows;
static int g_sms;

static double max_cycles()
{
    static long long h[1024];
    cudaMemcpy(h, g_cycles, sizeof(long long) * g_sms, cudaMemcpyDeviceToHost);
    long long m = 0;
    for (int i = 0; i < g_sms; i++) m = h[i] > m ? h[i] : m;
    return (double)m;
}

template <int OP>
static void run_pipe(const char *name, int iters = 2000)
{
    auto k = pipe_kernel<OP>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, TAB_SMEM);
    k<<<g_sms, 512, TAB_SMEM>>>(g_out, g_cycles, 50, g_rows);
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a);
    k<<<g_sms, 512, TAB_SMEM>>>(g_out, g_cycles, iters, g_rows);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    const double cyc = max_cycles();
    const Mix m = mix_of(OP);
    const double steps_per_warp = (double)iters * UNROLL * CH;
    const double warps = 512 / 32;
    const double per_clk = steps_per_warp * warps / cyc;    /* steps per clock per SM (warp granularity) */
    printf("{\"kind\": \"pipe\", \"name\": \"%s\", \"alu_per_step\": %d, \"fma_per_step\": %d, \"lsu_per_step\": %d, "
           "\"steps_per_clk_sm\": %.4f, \"alu_inst_per_clk_sm\": %.4f, \"fma_inst_per_clk_sm\": %.4f, "
           "\"lsu_inst_per_clk_sm\": %.4f, \"cycles\": %.0f, \"ms\": %.4f, \"sm_mhz_effective\": %.1f, \"err\": \"%s\"}\n",
           name, m.alu, m.fma, m.lsu, per_clk, per_clk * m.alu, per_clk * m.fma, per_clk * m.lsu, cyc, ms,
           cyc / (ms * 1e3), cudaGetErrorString(cudaGetLastError()));
}

template <int KIND, int MASK>
static void run_qr()
{
    auto k = qr_kernel<KIND, MASK>;
    const int iters = 4000;
    k<<<g_sms, 512>>>(g_out, g_cycles, 50);
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a);
    k<<<g_sms, 512>>>(g_out, g_cycles, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    const double cyc = max_cycles();
    const double qrs_per_warp = (double)iters * 4 * 4;
    const double per_clk = qrs_per_warp * (512 / 32) / cyc;
    printf("{\"kind\": \"quarter_round\", \"cipher\": \"%s\", \"fma_rot_mask\": %d, \"qr_per_clk_sm\": %.5f, "
           "\"clk_per_qr_sm\": %.3f, \"cycles\": %.0f, \"ms\": %.4f, \"err\": \"%s\"}\n",
           KIND == 0 ? "salsa20" : "chacha20", MASK, per_clk, 1.0 / per_clk, cyc, ms, cudaGetErrorString(cudaGetLastError()));
}

int main()
{
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    g_sms = p.multiProcessorCount;
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    printf("{\"kind\": \"device\", \"name\": \"%s\", \"sms\": %d, \"clock_mhz_nominal\": %.0f, \"warps_per_sm\": 16, "
           "\"chains_per_thread\": %d}\n", p.name, g_sms, khz / 1000.0, CH);
    cudaMalloc(&g_out, sizeof(uint32_t) * g_sms * 512);
    cudaMalloc(&g_cycles, sizeof(long long) * 1024);
    cudaMalloc(&g_rows, sizeof(uint4) * 4 * (ROWS_MASK + 1));
    cudaMemset(g_rows, 0x5a, sizeof(uint4) * 4 * (ROWS_MASK + 1));
    run_pipe<OP_LOP3>("LOP3");
    run_pipe<OP_SHF>("SHF");
    run_pipe<OP_PRMT>("PRMT");
    run_pipe<OP_IADD3>("IADD3");
    run_pipe<OP_IMAD>("IMAD");
    run_pipe<OP_IMADWIDE>("IMAD.WIDE+LOP3");
    run_pipe<OP_IMADHI>("IMAD.HI");
    run_pipe<OP_LDS>("PRMT+LDS.32 conflict-free");
    run_pipe<OP_LDS_LDG>("PRMT+LDS.32 + 3 broadcast LDG.128 per 128 LDS");
    run_pipe<OP_LDS_LDG_UNIT>("PRMT+LDS.32 + 16 broadcast LDG.128 per 1280 LDS");
    run_pipe<OP_LDS_MMA_UNIT>("PRMT+LDS.32 + 4 LDG.64, 24 PRMT, 10 IMMA.16816.U8 per 1280 LDS");
    run_pipe<OP_LDS_LDG64_UNIT>("PRMT+LDS.32 + 4 LDG.64, 24 PRMT, no IMMA per 1280 LDS");
    /* the same mixes 10x longer (about 22 ms), alternating: the rates are per SM clock, but what a
     * kernel costs is time, and sm_mhz_effective shows whether the clock moves with the mix */
    run_pipe<OP_LDS>("PRMT+LDS.32 conflict-free (long)", 20000);
    run_pipe<OP_LDS_LDG_UNIT>("PRMT+LDS.32 + 16 broadcast LDG.128 per 1280 LDS (long)", 20000);
    run_pipe<OP_LDS_MMA_UNIT>("PRMT+LDS.32 + 4 LDG.64, 24 PRMT, 10 IMMA.16816.U8 per 1280 LDS (long)", 20000);
    run_pipe<OP_LDS_LDG64_UNIT>("PRMT+LDS.32 + 4 LDG.64, 24 PRMT, no IMMA per 1280 LDS (long)", 20000);
    run_pipe<OP_LDS_LDG_UNIT>("PRMT+LDS.32 + 16 broadcast LDG.128 per 1280 LDS (long, again)", 20000);
    run_pipe<OP_MIX_LOP3_IMAD>("LOP3+IMAD");
    run_pipe<OP_MIX_LOP3_SHF_IMAD>("LOP3+SHF+IMAD");
    run_pipe<OP_MIX_LDS_PRMT_LOP3>("PRMT+LDS+LOP3");
    run_pipe<OP_MIX_LOP3_IMADWIDE>("LOP3+IMAD.WIDE+LOP3");
    run_qr<0, 0>(); run_qr<0, 1>(); run_qr<0, 2>(); run_qr<0, 4>(); run_qr<0, 8>(); run_qr<0, 5>(); run_qr<0, 10>();
    run_qr<0, 3>(); run_qr<0, 15>();
    run_qr<1, 0>(); run_qr<1, 1>(); run_qr<1, 2>(); run_qr<1, 4>(); run_qr<1, 8>(); run_qr<1, 5>(); run_qr<1, 10>();
    run_qr<1, 15>();
    printf("{\"kind\": \"end\", \"err\": \"%s\"}\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
