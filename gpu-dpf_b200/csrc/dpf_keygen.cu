/*
 * dpf_keygen.cu -- batched DPF key generation on the GPU (SURVEY.md section 8(f) rank 1, "optionally GPU").
 *
 * Key generation is the client's job in the protocol and stays a CPU function in the reference
 * (dpf_wrapper.cu:49-68 -> dpf_base/dpf.h:403-464); a benchmark or a load generator, however, needs
 * thousands of key pairs per batch (BASELINE config 5: 8192), and each costs ~6*depth PRF calls plus
 * its random draws.  One thread per key pair here, for every kind of key; the construction, the draw
 * order and the generator (ChaCha20, RFC 8439 block function, keyed by 44 bytes of caller entropy per
 * key) are exactly those of host::KeyBuilder (dpf_host.cpp: gen_secure, gen_leaves), so the two produce
 * bit-identical keys for identical seeds -- which is how tests/test_gpu_parity.py and
 * tests/test_gpu_group_gen_queries.py check it.
 *
 * Not a hot path: the payloads live in local memory, AES goes through a plain 1 KiB T-table in global
 * memory.  Each level's correction words are final once the level is built and go straight to the output.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "dpf_core.cuh"
#include "dpf_kernels.cuh"

namespace b200dpf {

namespace {

struct AesGlobalTable {
    const uint32_t *te0;   /* 256 entries of Te0 in global memory */
    template <int K, int BYTE>
    __device__ __forceinline__ uint32_t te(uint32_t word) const
    {
        const uint32_t v = __ldg(te0 + ((word >> (8 * BYTE)) & 0xffu));
        return K == 0 ? v : __funnelshift_l(v, v, 8 * K);
    }
};

__device__ __forceinline__ u128 to_u128(const Seed &s)
{
    return ((u128)s.w << 96) | ((u128)s.z << 64) | ((u128)s.y << 32) | (u128)s.x;
}
__device__ __forceinline__ Seed from_u128(u128 v)
{
    return make_seed((uint32_t)v, (uint32_t)(v >> 32), (uint32_t)(v >> 64), (uint32_t)(v >> 96));
}

template <int PRF>
__device__ __forceinline__ u128 prf128(const AesGlobalTable &ta, u128 seed, uint32_t pos)
{
    return to_u128(expand_one<PRF>(ta, from_u128(seed), pos));
}

/* ChaCha20 keystream as a deterministic random bit generator: same state layout and draw order as
 * host::ChaCha20Rng (dpf_host.cpp) */
struct ChaCha20Drbg {
    uint32_t state[16];
    uint32_t block[16];
    int used;

    __device__ void init(const uint8_t *key32, const uint8_t *nonce12)
    {
        state[0] = 0x61707865u; state[1] = 0x3320646eu; state[2] = 0x79622d32u; state[3] = 0x6b206574u;
        for (int i = 0; i < 8; i++)
            state[4 + i] = (uint32_t)key32[4 * i] | ((uint32_t)key32[4 * i + 1] << 8) | ((uint32_t)key32[4 * i + 2] << 16) |
                           ((uint32_t)key32[4 * i + 3] << 24);
        state[12] = 0;
        for (int i = 0; i < 3; i++)
            state[13 + i] = (uint32_t)nonce12[4 * i] | ((uint32_t)nonce12[4 * i + 1] << 8) |
                            ((uint32_t)nonce12[4 * i + 2] << 16) | ((uint32_t)nonce12[4 * i + 3] << 24);
        used = 16;
    }
    __device__ static void qr(uint32_t *x, int a, int b, int c, int d)
    {
        x[a] += x[b]; x[d] = __funnelshift_l(x[d] ^ x[a], x[d] ^ x[a], 16);
        x[c] += x[d]; x[b] = __funnelshift_l(x[b] ^ x[c], x[b] ^ x[c], 12);
        x[a] += x[b]; x[d] = __funnelshift_l(x[d] ^ x[a], x[d] ^ x[a], 8);
        x[c] += x[d]; x[b] = __funnelshift_l(x[b] ^ x[c], x[b] ^ x[c], 7);
    }
    __device__ void refill()
    {
        uint32_t x[16];
        for (int i = 0; i < 16; i++) x[i] = state[i];
        for (int r = 0; r < 10; r++) {
            qr(x, 0, 4, 8, 12); qr(x, 1, 5, 9, 13); qr(x, 2, 6, 10, 14); qr(x, 3, 7, 11, 15);
            qr(x, 0, 5, 10, 15); qr(x, 1, 6, 11, 12); qr(x, 2, 7, 8, 13); qr(x, 3, 4, 9, 14);
        }
        for (int i = 0; i < 16; i++) block[i] = x[i] + state[i];
        state[12]++;
        used = 0;
    }
    __device__ uint32_t draw32()
    {
        if (used == 16) refill();
        return block[used++];
    }
    __device__ u128 draw128()
    {
        u128 v = 0;
        for (int i = 0; i < 4; i++) v |= (u128)draw32() << (32 * i);
        return v;
    }
    __device__ u128 draw128_odd()
    {
        u128 k = 0;
        while ((k & 1) == 0) k = draw128();
        return k;
    }
};

__device__ __forceinline__ void store_slot(uint4 *key, int slot, u128 v)
{
    key[slot] = make_uint4((uint32_t)v, (uint32_t)(v >> 32), (uint32_t)(v >> 64), (uint32_t)(v >> 96));
}

/* correction word `row` of bank 2 (seed LSB set) or bank 1, without indexing the arrays at run time */
__device__ __forceinline__ u128 pick(const u128 *c1, const u128 *c2, bool bank2, int row)
{
    const u128 w1 = row ? c1[1] : c1[0], w2 = row ? c2[1] : c2[0];
    return bank2 ? w2 : w1;
}

/* Where a key pair goes: the two servers' keys at the same offset of out_a and out_b, and the slot of
 * correction word j (0..3) of level L and of the root in that layout.  Wire: the reference's 131 slots,
 * cw_1[2L + j] at 1 + 2L + j and cw_2[2L + j - 2] at 65 + 2L + j - 2.  Compact: the b200dpf_key_pack bytes,
 * level L's four words at 2 + 4L + j. */
struct KeyOut {
    uint4 *a, *b;
    bool compact;
    __device__ __forceinline__ int cw_slot(int L, int j) const
    {
        if (compact) return 2 + 4 * L + j;
        return (j < 2 ? 1 : 65 - 2) + 2 * L + j;
    }
    __device__ __forceinline__ void put(int slot, u128 va, u128 vb) const
    {
        store_slot(a, slot, va);
        store_slot(b, slot, vb);
    }
    /* level L's correction words c1[2], c2[2], the same for both servers */
    __device__ __forceinline__ void level(int L, const u128 *c1, const u128 *c2) const
    {
        for (int j = 0; j < 4; j++) {
            const u128 v = j < 2 ? c1[j] : c2[j - 2];
            put(cw_slot(L, j), v, v);
        }
    }
};

/*
 * The log(n) construction of dpf_base/dpf.h:403-464 (levels above the base) over the N = 2 base of
 * dpf.h:290-360, written as the two loops the reference's recursion unrolls into: on the way DOWN
 * every level draws the odd payload of the level below; at the bottom the two root seeds and the
 * base correction words are made; on the way UP every level derives its correction words from the
 * PRF values of the two seeds handed up from below.  Level 0 (the leaves' payload) adds in GROUP
 * (level0_add / level0_sub, as host::KeyBuilder<GROUP>), every other level in Z/2^128.
 *
 * Thread k makes one key pair.  A flat batch (bins == null): alphas[k], seeds44[k], every tree of depth p.depth.
 * A query batch of a grouped context: k = g * nq + q is key g of query q (bin-major, so a warp's threads
 * share a depth), with alphas / seeds [nq][nbins] and bins[g] = (uint4 offset of the key in a compact
 * query, tree depth of bin g).
 */
template <int PRF, int GROUP>
__global__ void __launch_bounds__(64, 1) keygen_kernel(const KeygenParams p)
{
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= p.count) return;
    AesGlobalTable ta;
    ta.te0 = p.te0;

    int64_t idx = k;   /* of the key's alpha and seed, and of the key pair in a wire-format output */
    int depth = p.depth;
    uint64_t off_v = (uint64_t)k * 131u;
    uint32_t rows = 0;   /* trimmed query batches: the bin's live rows */
    if (p.bins) {
        const uint32_t g = (uint32_t)(k / p.nq), q = (uint32_t)(k - (int64_t)g * p.nq);
        const uint2 b = p.bins[g];
        idx = (int64_t)q * p.nbins + g;
        depth = (int)b.y;
        off_v = p.compact ? (uint64_t)q * p.query_v + b.x : (uint64_t)idx * 131u;
        if (p.bin_place[g].depth == PLACE_IDENTITY) rows = p.bin_place[g].n;
    }
    const KeyOut out{p.out_a + off_v, p.out_b + off_v, p.compact != 0};

    /* the key for the low depth + lane_bits bits of alpha: its leaf, and the payload at level 0 (beta = 1,
     * dpf_wrapper.cu:53; early-terminated: lane alpha & 3 of the leaf; XOR-shared: bit alpha & 127) */
    uint64_t a_row = (uint64_t)p.alphas[idx];
    if (rows != 0) {   /* row r = alpha mod n_g of a trimmed bin */
        int64_t r = p.alphas[idx] % (int64_t)rows;
        if (r < 0) r += rows;
        a_row = trimmed_alpha((uint64_t)r, depth, p.lane_bits);
    }
    const uint64_t alpha = (a_row & ((((uint64_t)1) << (depth + p.lane_bits)) - 1u)) >> p.lane_bits;
    u128 beta[32];
    beta[0] = GROUP == GROUP_LANES32 ? (u128)1 << (32 * (a_row & 3u)) : GROUP == GROUP_XOR128 ? (u128)1 << (a_row & 127u) : (u128)1;

    ChaCha20Drbg g;
    g.init(p.seeds44 + 44 * idx, p.seeds44 + 44 * idx + 32);
    for (int L = 0; L + 1 < depth; L++) beta[L + 1] = g.draw128_odd();

    u128 up_a, up_b;
    {
        /* N = 2 base: one seed per server, differing in the LSB (dpf.h:318-331) */
        const int L = depth - 1;
        const int row = (int)(alpha & 1u);
        u128 ka = g.draw128(), kb = g.draw128();
        ka &= ~(u128)1;
        kb = (kb & ~(u128)1) | 1;
        out.put(p.compact ? 1 : 129, ka, kb);
        u128 delta[2], c1[2], c2[2];
        for (int i = 0; i < 2; i++) {
            const u128 fa = prf128<PRF>(ta, ka, (uint32_t)i), fb = prf128<PRF>(ta, kb, (uint32_t)i);
            delta[i] = L == 0 ? level0_sub<GROUP>(fa, fb) : fa - fb;
            if (i == row) delta[i] = L == 0 ? level0_sub<GROUP>(delta[i], beta[L]) : delta[i] - beta[L];
        }
        for (int i = 0; i < 2; i++) {
            c1[i] = g.draw128();
            c2[i] = L == 0 ? level0_add<GROUP>(c1[i], delta[i]) : c1[i] + delta[i];
        }
        out.level(L, c1, c2);
        up_a = prf128<PRF>(ta, ka, (uint32_t)row) + pick(c1, c2, (ka & 1) != 0, row);
        up_b = prf128<PRF>(ta, kb, (uint32_t)row) + pick(c1, c2, (kb & 1) != 0, row);
    }
    for (int L = depth - 2; L >= 0; L--) {
        const int row = (int)((alpha >> (depth - 1 - L)) & 1u);
        const bool a_even = (up_a & 1) == 0;
        u128 c1[2], c2[2];
        for (int i = 0; i < 2; i++) {
            const u128 fa = prf128<PRF>(ta, up_a, (uint32_t)i), fb = prf128<PRF>(ta, up_b, (uint32_t)i);
            u128 d = L == 0 ? level0_sub<GROUP>(fb, fa) : fb - fa;
            if (a_even) d = L == 0 ? level0_sub<GROUP>((u128)0, d) : (u128)0 - d;
            c1[i] = g.draw128();
            c2[i] = L == 0 ? level0_add<GROUP>(c1[i], d) : c1[i] + d;
            if (i == row) {
                if (L == 0) c1[i] = a_even ? level0_add<GROUP>(c1[i], beta[0]) : level0_sub<GROUP>(c1[i], beta[0]);
                else c1[i] += a_even ? beta[L] : (u128)0 - beta[L];
            }
        }
        out.level(L, c1, c2);
        if (L == 0) break;   /* the seeds below level 0 are the leaves: nothing is handed up */
        const u128 na = prf128<PRF>(ta, up_a, (uint32_t)row) + pick(c1, c2, (up_a & 1) != 0, row);
        const u128 nb = prf128<PRF>(ta, up_b, (uint32_t)row) + pick(c1, c2, (up_b & 1) != 0, row);
        up_a = na;
        up_b = nb;
    }

    if (p.compact) {
        /* b200dpf_key_pack's header: magic, depth, zeros; nothing past the key's own levels */
        out.put(0, (u128)p.magic | ((u128)(uint32_t)depth << 32), (u128)p.magic | ((u128)(uint32_t)depth << 32));
        return;
    }
    /* the reference's wire format, dpf_wrapper.cu:26-35: slot 0 = (depth, lane_bits, 0, 0), slot 130 = n,
     * the correction words of the levels below the tree zero */
    const u128 head = (u128)(uint32_t)depth | ((u128)(uint32_t)p.lane_bits << 32);
    out.put(0, head, head);
    for (int s = 2 * depth; s < 64; s++) {
        out.put(1 + s, 0, 0);
        out.put(65 + s, 0, 0);
    }
    const u128 n = (u128)1 << (depth + p.lane_bits);
    out.put(130, n, n);
}

template <int GROUP>
cudaError_t launch_group(int prf, const KeygenParams &p, int grid, cudaStream_t stream)
{
    switch (prf) {
    case PRF_DUMMY: keygen_kernel<PRF_DUMMY, GROUP><<<grid, 64, 0, stream>>>(p); break;
    case PRF_SALSA20: keygen_kernel<PRF_SALSA20, GROUP><<<grid, 64, 0, stream>>>(p); break;
    case PRF_CHACHA20: keygen_kernel<PRF_CHACHA20, GROUP><<<grid, 64, 0, stream>>>(p); break;
    case PRF_AES128: keygen_kernel<PRF_AES128, GROUP><<<grid, 64, 0, stream>>>(p); break;
    default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_keygen(int prf, int group, const KeygenParams &p, cudaStream_t stream)
{
    if (p.count <= 0) return cudaSuccess;
    const int grid = (int)((p.count + 63) / 64);
    switch (group) {
    case GROUP_ADD128: return launch_group<GROUP_ADD128>(prf, p, grid, stream);
    case GROUP_LANES32: return launch_group<GROUP_LANES32>(prf, p, grid, stream);
    case GROUP_XOR128: return launch_group<GROUP_XOR128>(prf, p, grid, stream);
    default: return cudaErrorInvalidValue;
    }
}

}  // namespace b200dpf
