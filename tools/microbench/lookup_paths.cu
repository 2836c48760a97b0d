// Microbenchmark: how many per-lane random 32-bit table lookups per clock per SM can each
// on-chip path sustain, alone and combined with conflict-free shared-memory lookups?
//   S: shared memory, table replicated per bank (lane L reads bank L)       -- what the AES kernel uses
//   C: constant memory, per-lane (divergent) index
//   G: global memory through L1 (1 KiB table, ld.global.nc), per-lane index
//   T: texture object fetch (tex1Dfetch), per-lane index
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o bin/lookup_paths lookup_paths.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__constant__ uint32_t c_tab[256];

template <int NS, int NC, int NG, int NT>
__global__ void __launch_bounds__(384, 1) k(const uint32_t *g_tab, cudaTextureObject_t tex, uint32_t *out, int iters)
{
    extern __shared__ uint32_t s_tab[];   // [256][32]
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x) s_tab[i] = c_tab[i >> 5] ^ (i & 31);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    uint32_t x0 = threadIdx.x * 2654435761u + blockIdx.x, x1 = x0 ^ 0x9e3779b9u, x2 = x0 * 3, x3 = ~x0;
    uint32_t acc = 0;
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            uint32_t v = 0;
            uint32_t xs[4] = {x0, x1, x2, x3};
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const uint32_t x = xs[q];
                if (NS > q) v ^= s_tab[((x >> (8 * j)) & 255) * 32 + lane];
                if (NC > q) v ^= c_tab[(x >> (8 * j + 1)) & 255];
                if (NG > q) v ^= __ldg(g_tab + ((x >> (8 * j + 2)) & 255));
                if (NT > q) v ^= tex1Dfetch<uint32_t>(tex, (int)((x >> (8 * j + 3)) & 255));
            }
            acc += v;
        }
        x0 = x0 * 1664525u + acc; x1 = x1 * 22695477u + x0; x2 ^= x1 >> 3; x3 += x2;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <int NS, int NC, int NG, int NT>
void run(const char *name, const uint32_t *g_tab, cudaTextureObject_t tex, uint32_t *out, int sms, double mhz)
{
    auto kern = k<NS, NC, NG, NT>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768);
    const int iters = 20000;
    kern<<<sms, 384, 32768>>>(g_tab, tex, out, 100);
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a);
    kern<<<sms, 384, 32768>>>(g_tab, tex, out, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    const double lookups_per_thread = (double)iters * 4 * (NS + NC + NG + NT);
    const double per_clk_sm = lookups_per_thread * 384 / (ms * 1e-3 * mhz * 1e6);
    printf("%-28s S=%d C=%d G=%d T=%d  %8.3f ms  %7.2f lookups/clk/SM  (smem part %.2f)\n", name, NS, NC, NG, NT, ms,
           per_clk_sm, per_clk_sm * NS / (NS + NC + NG + NT));
}

int main()
{
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int khz = 0;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    const double mhz = khz / 1000.0;
    printf("%s, %d SMs, %.0f MHz nominal\n", p.name, p.multiProcessorCount, mhz);
    uint32_t h[256];
    for (int i = 0; i < 256; i++) h[i] = i * 2654435761u;
    cudaMemcpyToSymbol(c_tab, h, sizeof h);
    uint32_t *g_tab, *out;
    cudaMalloc(&g_tab, sizeof h);
    cudaMemcpy(g_tab, h, sizeof h, cudaMemcpyHostToDevice);
    cudaMalloc(&out, (size_t)p.multiProcessorCount * 384 * 4 * 4);
    cudaResourceDesc rd = {};
    rd.resType = cudaResourceTypeLinear;
    rd.res.linear.devPtr = g_tab;
    rd.res.linear.desc = cudaCreateChannelDesc<uint32_t>();
    rd.res.linear.sizeInBytes = sizeof h;
    cudaTextureDesc td = {};
    td.readMode = cudaReadModeElementType;
    cudaTextureObject_t tex;
    cudaCreateTextureObject(&tex, &rd, &td, nullptr);
    const int sms = p.multiProcessorCount;
    run<4, 0, 0, 0>("smem only", g_tab, tex, out, sms, mhz);
    run<0, 4, 0, 0>("const only", g_tab, tex, out, sms, mhz);
    run<0, 0, 4, 0>("global/L1 only", g_tab, tex, out, sms, mhz);
    run<0, 0, 0, 4>("texture only", g_tab, tex, out, sms, mhz);
    run<4, 1, 0, 0>("smem x4 + const x1", g_tab, tex, out, sms, mhz);
    run<4, 0, 1, 0>("smem x4 + global x1", g_tab, tex, out, sms, mhz);
    run<4, 0, 0, 1>("smem x4 + texture x1", g_tab, tex, out, sms, mhz);
    run<3, 0, 0, 1>("smem x3 + texture x1", g_tab, tex, out, sms, mhz);
    run<3, 1, 0, 0>("smem x3 + const x1", g_tab, tex, out, sms, mhz);
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
