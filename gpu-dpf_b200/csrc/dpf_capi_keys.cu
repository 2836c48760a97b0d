/*
 * dpf_capi_keys.cu -- the key entry points of the C ABI: generation on the CPU and the GPU, CPU evaluation, and the
 * compact key format, for every kind of key.
 */
#include "dpf_ctx.h"

#include <cstdio>

namespace {

/* The CPU entry points of every kind of key; `name` is the entry point's, without "b200dpf_", in messages. */

/* The refusal of entry point `name` of a key that is not of `kind` */
int fail_not_kind(int kind, const char *name)
{
    if (kind == host::KIND_STANDARD) return fail(B200DPF_EINVAL, "%s: malformed key", name);
    return fail(B200DPF_EINVAL, "%s: not an %s key", name, host::kKinds[kind].name);
}

/* one key pair from the ChaCha20 DRBG: b200dpf_gen_secure for standard keys */
int gen_drbg_one(int kind, int64_t alpha, int64_t n, const uint8_t *seed, int prf, int32_t *key_a, int32_t *key_b)
{
    if (kind == host::KIND_STANDARD) return host::gen_secure(alpha, n, seed, prf, key_a, key_b);
    return host::gen_leaves(kind, alpha, n, seed, prf, key_a, key_b);
}

int gen_drbg(int kind, const char *name, int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf,
             int32_t *key_a, int32_t *key_b)
{
    const host::KindInfo &k = host::kKinds[kind];
    if (!key_a || !key_b) return fail(B200DPF_EINVAL, "null key buffer");
    if (!seed || seed_len < 44) return fail(B200DPF_EINVAL, "%s needs at least 44 bytes of seed (got %zu)", name, seed_len);
    if (gen_drbg_one(kind, alpha, n, seed, prf, key_a, key_b) != 0)
        return fail(B200DPF_EINVAL, "%s: need power-of-two n in [%lld, 2^%d], 0 <= alpha < n, valid prf (alpha=%lld n=%lld prf=%d)",
                    name, (long long)k.n_min, ilog2(k.n_max), (long long)alpha, (long long)n, prf);
    return B200DPF_OK;
}

int gen_batch_drbg(int kind, const char *name, const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                   int nthreads, int32_t *keys_a, int32_t *keys_b)
{
    if (!alphas || !seeds44 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad %s argument", name);
    if (!gen_parallel(count, nthreads, [&](int64_t i) {
            return gen_drbg_one(kind, alphas[i], n, seeds44 + 44 * i, prf, keys_a + i * host::KEY_WORDS, keys_b + i * host::KEY_WORDS);
        }))
        return fail(B200DPF_EINVAL, "%s: invalid alpha/n/prf in batch", name);
    return B200DPF_OK;
}

/* gen_batch_drbg on a GPU (b200dpf_gen_batch_gpu, _et, _xor): host alphas and seeds, keys to host or device
 * memory; `cpu_name` is the CPU entry point of the same keys, named when there is no device */
int gen_batch_gpu_kind(int kind, const char *name, const char *cpu_name, const int64_t *alphas, const uint8_t *seeds44,
                       int64_t count, int64_t n, int prf, int device, int32_t *keys_a, int32_t *keys_b)
{
    const host::KindInfo &k = host::kKinds[kind];
    if (!alphas || !seeds44 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad %s argument", name);
    if (n < k.n_min || n > k.n_max || (n & (n - 1)) != 0)
        return fail(B200DPF_EINVAL, "n=%lld must be a power of two in [%lld, 2^%d]", (long long)n, (long long)k.n_min, ilog2(k.n_max));
    if (prf < B200DPF_PRF_DUMMY || prf > B200DPF_PRF_AES128) return fail(B200DPF_EINVAL, "unknown prf id %d", prf);
    for (int64_t i = 0; i < count; i++)
        if (alphas[i] < 0 || alphas[i] >= n) return fail(B200DPF_EINVAL, "%s: alpha[%lld]=%lld out of range", name, (long long)i, (long long)alphas[i]);
    if (count == 0) return B200DPF_OK;
    std::optional<DeviceGuard> guard;
    char hint[64];
    snprintf(hint, sizeof hint, "use b200dpf_%s on the CPU", cpu_name);
    int rc = open_device(device, hint, &guard);
    if (rc) return rc;
    const size_t key_bytes = (size_t)count * kKeyBytes;
    DeviceBuffer<int64_t> d_alphas;
    DeviceBuffer<uint8_t> d_seeds;
    DeviceBuffer<uint32_t> d_te0;
    DeviceBuffer<uint4> d_a, d_b;
    rc = d_alphas.reserve((size_t)count * sizeof(int64_t));
    if (!rc) rc = d_seeds.reserve((size_t)count * 44);
    if (!rc) rc = d_te0.reserve(256 * sizeof(uint32_t));
    if (!rc) rc = d_a.reserve(key_bytes);
    if (!rc) rc = d_b.reserve(key_bytes);
    if (rc) return rc;
    cudaError_t e = cudaMemcpy(d_alphas.ptr, alphas, (size_t)count * sizeof(int64_t), cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(d_seeds.ptr, seeds44, (size_t)count * 44, cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(d_te0.ptr, host::aes_te0(), 256 * sizeof(uint32_t), cudaMemcpyHostToDevice);
    KeygenParams p{};
    p.alphas = d_alphas.ptr;
    p.seeds44 = d_seeds.ptr;
    p.count = count;
    p.depth = ilog2(n) - k.lane_bits;
    p.lane_bits = k.lane_bits;
    p.te0 = d_te0.ptr;
    p.out_a = d_a.ptr;
    p.out_b = d_b.ptr;
    if (e == cudaSuccess) e = launch_keygen(prf, k.group, p, nullptr);
    if (e == cudaSuccess) e = cudaMemcpy(keys_a, d_a.ptr, key_bytes, cudaMemcpyDefault);      /* host or device destination */
    if (e == cudaSuccess) e = cudaMemcpy(keys_b, d_b.ptr, key_bytes, cudaMemcpyDefault);
    if (e != cudaSuccess) return fail(B200DPF_ECUDA, "%s: %s", name, cudaGetErrorString(e));
    return B200DPF_OK;
}

int eval_cpu_kind(int kind, const char *name, const int32_t *key, int prf, int32_t *out)
{
    if (!key || !out) return fail(B200DPF_EINVAL, "null buffer");
    const int rc = host::eval_cpu(key, kind, prf, out);
    if (rc == -1) return fail_not_kind(kind, name);
    if (rc) return fail(B200DPF_EINVAL, "%s: unknown prf id %d", name, prf);
    return B200DPF_OK;
}

int key_pack_kind(int kind, const char *name, const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    if (!key || !out) return fail(B200DPF_EINVAL, "null buffer");
    const int depth = host::key_depth(key, kind);
    if (depth < 1 || host::key_n(key, kind) < 0) return fail_not_kind(kind, name);
    const size_t need = b200dpf_key_packed_size(depth);
    if (out_cap < need) return fail(B200DPF_EINVAL, "%s: need %zu bytes, have %zu", name, need, out_cap);
    pack_compact(key, out, depth, host::kKinds[kind].magic);
    if (written) *written = need;
    return B200DPF_OK;
}

int key_unpack_kind(int kind, const char *name, const uint8_t *in, size_t in_len, int32_t *key)
{
    const host::KindInfo &k = host::kKinds[kind];
    if (!in || !key) return fail(B200DPF_EINVAL, "null buffer");
    if (in_len < 32 || std::memcmp(in, k.magic, 4) != 0) return fail(B200DPF_EINVAL, "%s: bad header", name);
    const int depth = in[4];
    bool pad_zero = true;
    for (int i = 5; i < 16; i++) pad_zero = pad_zero && in[i] == 0;
    if (depth < 1 || depth > k.max_depth || !pad_zero || in_len != b200dpf_key_packed_size(depth))
        return fail(B200DPF_EINVAL, "%s: depth %d does not match %zu bytes", name, depth, in_len);
    std::memset(key, 0, sizeof(int32_t) * host::KEY_WORDS);
    uint8_t *kb = reinterpret_cast<uint8_t *>(key);
    kb[16 * host::SLOT_DEPTH] = (uint8_t)depth;
    kb[16 * host::SLOT_DEPTH + 4] = (uint8_t)k.lane_bits;
    std::memcpy(kb + 16 * host::SLOT_ROOT, in + 16, 16);
    for (int L = 0; L < depth; L++) {
        const uint8_t *o = in + 32 + 64 * L;
        std::memcpy(kb + 16 * (host::SLOT_CW1 + 2 * L), o, 32);
        std::memcpy(kb + 16 * (host::SLOT_CW2 + 2 * L), o + 32, 32);
    }
    const uint64_t n = (uint64_t)1 << (depth + k.lane_bits);
    std::memcpy(kb + 16 * host::SLOT_N, &n, 8);
    return B200DPF_OK;
}

}  // namespace

extern "C" {

int b200dpf_gen(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf,
                int32_t *key_a, int32_t *key_b)
{
    if (!key_a || !key_b) return fail(B200DPF_EINVAL, "null key buffer");
    uint32_t seed32 = 0;
    for (size_t i = 0; i < 4 && i < seed_len && seed; i++) seed32 |= (uint32_t)seed[i] << (8 * i);
    if (host::gen(alpha, n, seed32, prf, key_a, key_b) != 0)
        return fail(B200DPF_EINVAL, "gen: need power-of-two n >= 2, 0 <= alpha < n, valid prf (alpha=%lld n=%lld prf=%d)",
                    (long long)alpha, (long long)n, prf);
    return B200DPF_OK;
}

int b200dpf_gen_secure(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf,
                       int32_t *key_a, int32_t *key_b)
{
    return gen_drbg(host::KIND_STANDARD, "gen_secure", alpha, n, seed, seed_len, prf, key_a, key_b);
}

int b200dpf_gen_batch(const int64_t *alphas, const uint32_t *seeds32, int64_t count, int64_t n, int prf,
                      int nthreads, int32_t *keys_a, int32_t *keys_b)
{
    if (!alphas || !seeds32 || !keys_a || !keys_b || count < 0) return fail(B200DPF_EINVAL, "bad gen_batch argument");
    if (!gen_parallel(count, nthreads, [&](int64_t i) {
            return host::gen(alphas[i], n, seeds32[i], prf, keys_a + i * host::KEY_WORDS, keys_b + i * host::KEY_WORDS);
        }))
        return fail(B200DPF_EINVAL, "gen_batch: invalid alpha/n/prf in batch");
    return B200DPF_OK;
}

int b200dpf_gen_batch_secure(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf,
                             int nthreads, int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_drbg(host::KIND_STANDARD, "gen_batch_secure", alphas, seeds44, count, n, prf, nthreads, keys_a, keys_b);
}

int b200dpf_gen_batch_gpu(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int device,
                          int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_gpu_kind(host::KIND_STANDARD, "gen_batch_gpu", "gen_batch_secure", alphas, seeds44, count, n, prf, device,
                              keys_a, keys_b);
}

int b200dpf_eval_cpu(const int32_t *key, int prf, int32_t *out_n)
{
    return eval_cpu_kind(host::KIND_STANDARD, "eval_cpu", key, prf, out_n);
}

size_t b200dpf_key_packed_size(int depth) { return depth >= 1 && depth <= 32 ? (size_t)32 + 64u * (size_t)depth : 0; }

int b200dpf_key_pack(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    return key_pack_kind(host::KIND_STANDARD, "key_pack", key, out, out_cap, written);
}

int b200dpf_key_unpack(const uint8_t *in, size_t in_len, int32_t *key)
{
    return key_unpack_kind(host::KIND_STANDARD, "key_unpack", in, in_len, key);
}

int64_t b200dpf_key_n(const int32_t *key) { return key ? host::key_n(key, host::KIND_STANDARD) : -1; }
int b200dpf_key_depth(const int32_t *key) { return key ? host::key_depth(key, host::KIND_STANDARD) : -1; }

/* ---- early-terminated keys ---- */

int b200dpf_gen_et(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf, int32_t *key_a, int32_t *key_b)
{
    return gen_drbg(host::KIND_ET, "gen_et", alpha, n, seed, seed_len, prf, key_a, key_b);
}

int b200dpf_gen_batch_et(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int nthreads,
                         int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_drbg(host::KIND_ET, "gen_batch_et", alphas, seeds44, count, n, prf, nthreads, keys_a, keys_b);
}

int b200dpf_gen_batch_gpu_et(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int device,
                             int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_gpu_kind(host::KIND_ET, "gen_batch_gpu_et", "gen_batch_et", alphas, seeds44, count, n, prf, device, keys_a,
                              keys_b);
}

int b200dpf_eval_cpu_et(const int32_t *key, int prf, int32_t *out_n)
{
    return eval_cpu_kind(host::KIND_ET, "eval_cpu_et", key, prf, out_n);
}

int b200dpf_key_pack_et(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    return key_pack_kind(host::KIND_ET, "key_pack_et", key, out, out_cap, written);
}

int b200dpf_key_unpack_et(const uint8_t *in, size_t in_len, int32_t *key)
{
    return key_unpack_kind(host::KIND_ET, "key_unpack_et", in, in_len, key);
}

/* ---- XOR-shared keys ---- */

int b200dpf_gen_xor(int64_t alpha, int64_t n, const uint8_t *seed, size_t seed_len, int prf, int32_t *key_a, int32_t *key_b)
{
    return gen_drbg(host::KIND_XOR, "gen_xor", alpha, n, seed, seed_len, prf, key_a, key_b);
}

int b200dpf_gen_batch_xor(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int nthreads,
                          int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_drbg(host::KIND_XOR, "gen_batch_xor", alphas, seeds44, count, n, prf, nthreads, keys_a, keys_b);
}

int b200dpf_gen_batch_gpu_xor(const int64_t *alphas, const uint8_t *seeds44, int64_t count, int64_t n, int prf, int device,
                              int32_t *keys_a, int32_t *keys_b)
{
    return gen_batch_gpu_kind(host::KIND_XOR, "gen_batch_gpu_xor", "gen_batch_xor", alphas, seeds44, count, n, prf, device, keys_a,
                              keys_b);
}

int b200dpf_eval_cpu_xor(const int32_t *key, int prf, uint32_t *bits)
{
    return eval_cpu_kind(host::KIND_XOR, "eval_cpu_xor", key, prf, reinterpret_cast<int32_t *>(bits));
}

int b200dpf_key_pack_xor(const int32_t *key, uint8_t *out, size_t out_cap, size_t *written)
{
    return key_pack_kind(host::KIND_XOR, "key_pack_xor", key, out, out_cap, written);
}

int b200dpf_key_unpack_xor(const uint8_t *in, size_t in_len, int32_t *key)
{
    return key_unpack_kind(host::KIND_XOR, "key_unpack_xor", in, in_len, key);
}

}  // extern "C"
