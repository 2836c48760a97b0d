/*
 * dpf_cpp_ext.cpp -- the `dpf_cpp` PyTorch extension module.
 *
 * Same pybind surface as the reference's dpf_wrapper.cu:188-204 (five
 * functions, six integer attributes, same argument order and types, results as
 * CPU int32 tensors), so the reference's dpf.py / sample.py / benchmark.py run
 * against it unchanged.  All work is delegated to the C ABI in
 * include/b200dpf.h; this file only converts tensors to pointers.
 *
 * Differences from the reference module, all additive:
 *   - eval_init accepts any entry size and any dtype; eval_gpu accepts any
 *     number of keys (the reference asserts 16 columns and exactly 512 keys);
 *   - errors surface as Python exceptions (RuntimeError) instead of assert /
 *     exit (dpf_wrapper.cu:7-15);
 *   - extra entry points: gen_batch, eval_gpu_packed, eval_init_sharded,
 *     expand_gpu, update_rows, version; attribute NATIVE_SHAPES = 1 advertises them.
 */
#include <torch/extension.h>
#include <torch/csrc/autograd/python_variable.h>

#include <ATen/detail/CUDAHooksInterface.h>

#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <functional>
#include <vector>

#include "b200dpf.h"

namespace {

constexpr int kKeyWords = B200DPF_KEY_WORDS;

void check(int rc, const char *what)
{
    if (rc != B200DPF_OK) throw std::runtime_error(std::string(what) + ": " + b200dpf_last_error());
}

b200dpf_ctx *ctx_of(const std::vector<void *> &buffers)
{
    if (buffers.empty() || buffers[0] == nullptr) throw std::runtime_error("dpf_cpp: empty buffer list (call eval_init first)");
    return static_cast<b200dpf_ctx *>(buffers[0]);
}

const int32_t *key_ptr(const at::Tensor &key)
{
    TORCH_CHECK(key.device().is_cpu(), "dpf_cpp: keys must be CPU tensors");
    TORCH_CHECK(key.scalar_type() == at::kInt && key.numel() == kKeyWords && key.is_contiguous(),
                "dpf_cpp: a key is a contiguous int32 tensor of 524 elements");
    return key.data_ptr<int32_t>();
}

/* The kinds of key (include/b200dpf.h): log2 table rows per leaf and maximum depth.  A key is slot 0 =
 * (d, lane_bits, 0, 0), 1 <= d <= max_depth, slot 130 = 2^(d + lane_bits) as a u64. */
struct KeyKind {
    int lane_bits, max_depth;
};
constexpr KeyKind kStandard{0, 32}, kEarlyTerminated{2, 29}, kXorShared{7, 24};

/* rows of a key of `kind`, or -1 */
int64_t key_rows(const int32_t *k, const KeyKind &kind)
{
    const uint32_t *w = reinterpret_cast<const uint32_t *>(k);
    if (w[1] != (uint32_t)kind.lane_bits || w[2] || w[3] || w[0] < 1 || w[0] > (uint32_t)kind.max_depth) return -1;
    const uint64_t n = (uint64_t)w[4 * 130] | (uint64_t)w[4 * 130 + 1] << 32;
    return n == (uint64_t)1 << (w[0] + kind.lane_bits) && !w[4 * 130 + 2] && !w[4 * 130 + 3] ? (int64_t)n : -1;
}

/* One helper per operation; `what` names the Python function in errors.  dpf_wrapper.cu:49-68 is gen. */
std::vector<at::Tensor> gen_with(int (*fn)(int64_t, int64_t, const uint8_t *, size_t, int, int32_t *, int32_t *),
                                 const char *what, int64_t k, int64_t n, const std::string &seed, int prf)
{
    at::Tensor a = torch::zeros({kKeyWords}, at::kInt);
    at::Tensor b = torch::zeros({kKeyWords}, at::kInt);
    check(fn(k, n, reinterpret_cast<const uint8_t *>(seed.data()), seed.size(), prf, a.data_ptr<int32_t>(), b.data_ptr<int32_t>()),
          what);
    return {a, b};
}

/* batched keygen from the ChaCha20 DRBG: seeds = 44 bytes of entropy per key, concatenated */
std::vector<at::Tensor> gen_batch_with(int (*fn)(const int64_t *, const uint8_t *, int64_t, int64_t, int, int, int32_t *, int32_t *),
                                       const char *what, const at::Tensor &alphas, int64_t n, const std::string &seeds, int prf,
                                       int nthreads)
{
    at::Tensor al = alphas.to(at::kLong).contiguous().cpu();
    TORCH_CHECK(al.dim() == 1 && (int64_t)seeds.size() == 44 * al.numel(), what, ": need 44 seed bytes per key");
    const int64_t count = al.numel();
    at::Tensor a = torch::zeros({count, kKeyWords}, at::kInt);
    at::Tensor b = torch::zeros({count, kKeyWords}, at::kInt);
    {
        py::gil_scoped_release nogil;
        check(fn(al.data_ptr<int64_t>(), reinterpret_cast<const uint8_t *>(seeds.data()), count, n, prf, nthreads,
                 a.data_ptr<int32_t>(), b.data_ptr<int32_t>()),
              what);
    }
    return {a, b};
}

/* the key's share of every row: int32 [n], or (XOR-shared keys, out_shift = 5) its share bits packed 32 per
 * int32, row i = bit (i & 31) of word i >> 5.  dpf_wrapper.cu:70-84 is eval_cpu. */
template <class Out>
at::Tensor eval_cpu_with(int (*fn)(const int32_t *, int, Out *), const char *what, const KeyKind &kind, int out_shift,
                         const char *not_kind, const at::Tensor &key, int prf)
{
    const int32_t *k = key_ptr(key);
    const int64_t n = key_rows(k, kind);
    TORCH_CHECK(n > 0, what, ": ", not_kind);
    at::Tensor result = torch::empty({n >> out_shift}, at::kInt);
    check(fn(k, prf, reinterpret_cast<Out *>(result.data_ptr<int32_t>())), what);
    return result;
}

/* compact wire form: int32[524] key tensor <-> bytes (32 + 64*depth) */
py::bytes key_pack_with(int (*fn)(const int32_t *, uint8_t *, size_t, size_t *), const char *what, const at::Tensor &key)
{
    const int32_t *k = key_ptr(key);
    std::string buf(b200dpf_key_packed_size(32), '\0');
    size_t written = 0;
    check(fn(k, reinterpret_cast<uint8_t *>(&buf[0]), buf.size(), &written), what);
    return py::bytes(buf.data(), written);
}

at::Tensor key_unpack_with(int (*fn)(const uint8_t *, size_t, int32_t *), const char *what, const std::string &packed)
{
    at::Tensor key = torch::zeros({kKeyWords}, at::kInt);
    check(fn(reinterpret_cast<const uint8_t *>(packed.data()), packed.size(), key.data_ptr<int32_t>()), what);
    return key;
}

std::vector<void *> eval_init_with(int (*fn)(b200dpf_ctx **, const int32_t *, int64_t, int, int, int, int), const char *what,
                                   const at::Tensor &table, int device, int shard_rank, int shard_count)
{
    TORCH_CHECK(table.dim() == 2, what, ": table must be [num_entries, entry_size]");
    /* dpf_wrapper.cu:107 converts each element with item<int>(); one vectorised cast here */
    at::Tensor t = table.to(at::kInt).contiguous();
    b200dpf_ctx *ctx = nullptr;
    check(fn(&ctx, t.data_ptr<int32_t>(), t.size(0), (int)t.size(1), device, shard_rank, shard_count), what);
    return {static_cast<void *>(ctx)};
}

/* batched keygen: alphas int64[B], seeds int64[B] (low 32 bits used) -> two int32[B,524] tensors */
std::vector<at::Tensor> gen_batch(const at::Tensor &alphas, int64_t n, const at::Tensor &seeds, int prf, int nthreads)
{
    at::Tensor al = alphas.to(at::kLong).contiguous().cpu();
    at::Tensor sd = seeds.to(at::kLong).contiguous().cpu();
    TORCH_CHECK(al.dim() == 1 && sd.sizes() == al.sizes(), "gen_batch: alphas and seeds are 1-D of equal length");
    const int64_t count = al.numel();
    std::vector<uint32_t> s32((size_t)count);
    for (int64_t i = 0; i < count; i++) s32[(size_t)i] = (uint32_t)sd.data_ptr<int64_t>()[i];
    at::Tensor a = torch::zeros({count, kKeyWords}, at::kInt);
    at::Tensor b = torch::zeros({count, kKeyWords}, at::kInt);
    {
        py::gil_scoped_release nogil;
        check(b200dpf_gen_batch(al.data_ptr<int64_t>(), s32.data(), count, n, prf, nthreads, a.data_ptr<int32_t>(),
                                b.data_ptr<int32_t>()),
              "gen_batch");
    }
    return {a, b};
}

using Keys = std::vector<at::Tensor>;
using Ctx = std::vector<void *>;

Keys gen(int64_t k, int64_t n, const std::string &seed, int prf) { return gen_with(b200dpf_gen, "gen", k, n, seed, prf); }
at::Tensor eval_cpu(const at::Tensor &key, int prf)
{
    return eval_cpu_with(b200dpf_eval_cpu, "eval_cpu", kStandard, 0, "malformed key", key, prf);
}
py::bytes key_pack(const at::Tensor &key) { return key_pack_with(b200dpf_key_pack, "key_pack", key); }
at::Tensor key_unpack(const std::string &packed) { return key_unpack_with(b200dpf_key_unpack, "key_unpack", packed); }
Keys gen_secure(int64_t k, int64_t n, const std::string &seed, int prf) { return gen_with(b200dpf_gen_secure, "gen_secure", k, n, seed, prf); }
Keys gen_batch_secure(const at::Tensor &alphas, int64_t n, const std::string &seeds, int prf, int nthreads)
{
    return gen_batch_with(b200dpf_gen_batch_secure, "gen_batch_secure", alphas, n, seeds, prf, nthreads);
}
Ctx eval_init_sharded(const at::Tensor &table, int device, int shard_rank, int shard_count)
{
    return eval_init_with(b200dpf_create, "eval_init", table, device, shard_rank, shard_count);
}

/* early-terminated keys: four table rows per tree leaf (include/b200dpf.h, b200dpf_gen_et) */
Keys gen_et(int64_t k, int64_t n, const std::string &seed, int prf) { return gen_with(b200dpf_gen_et, "gen_et", k, n, seed, prf); }
Keys gen_batch_et(const at::Tensor &alphas, int64_t n, const std::string &seeds, int prf, int nthreads)
{
    return gen_batch_with(b200dpf_gen_batch_et, "gen_batch_et", alphas, n, seeds, prf, nthreads);
}
at::Tensor eval_cpu_et(const at::Tensor &key, int prf)
{
    return eval_cpu_with(b200dpf_eval_cpu_et, "eval_cpu_et", kEarlyTerminated, 0, "not an early-terminated key", key, prf);
}
py::bytes key_pack_et(const at::Tensor &key) { return key_pack_with(b200dpf_key_pack_et, "key_pack_et", key); }
at::Tensor key_unpack_et(const std::string &packed) { return key_unpack_with(b200dpf_key_unpack_et, "key_unpack_et", packed); }
Ctx eval_init_et(const at::Tensor &table, int device, int shard_rank, int shard_count)
{
    return eval_init_with(b200dpf_create_et, "eval_init_et", table, device, shard_rank, shard_count);
}

/* XOR-shared keys: 128 table rows per tree leaf, results XOR (include/b200dpf.h, b200dpf_gen_xor) */
Keys gen_xor(int64_t k, int64_t n, const std::string &seed, int prf) { return gen_with(b200dpf_gen_xor, "gen_xor", k, n, seed, prf); }
Keys gen_batch_xor(const at::Tensor &alphas, int64_t n, const std::string &seeds, int prf, int nthreads)
{
    return gen_batch_with(b200dpf_gen_batch_xor, "gen_batch_xor", alphas, n, seeds, prf, nthreads);
}
at::Tensor eval_cpu_xor(const at::Tensor &key, int prf)
{
    return eval_cpu_with(b200dpf_eval_cpu_xor, "eval_cpu_xor", kXorShared, 5, "not an XOR-shared key", key, prf);
}
py::bytes key_pack_xor(const at::Tensor &key) { return key_pack_with(b200dpf_key_pack_xor, "key_pack_xor", key); }
at::Tensor key_unpack_xor(const std::string &packed) { return key_unpack_with(b200dpf_key_unpack_xor, "key_unpack_xor", packed); }
Ctx eval_init_xor(const at::Tensor &table, int device, int shard_rank, int shard_count)
{
    return eval_init_with(b200dpf_create_xor, "eval_init_xor", table, device, shard_rank, shard_count);
}

/* one table on several GPUs of this process (b200dpf_create_multi); axis: 0 auto, 1 entries, 2 keys */
std::vector<void *> eval_init_multi(const at::Tensor &table, const std::vector<int> &devices, int axis)
{
    TORCH_CHECK(table.dim() == 2, "eval_init: table must be [num_entries, entry_size]");
    TORCH_CHECK(!devices.empty(), "eval_init_multi: empty device list");
    at::Tensor t = table.to(at::kInt).contiguous().cpu();
    b200dpf_ctx *ctx = nullptr;
    {
        py::gil_scoped_release nogil;
        check(b200dpf_create_multi(&ctx, t.data_ptr<int32_t>(), t.size(0), (int)t.size(1), devices.data(), (int)devices.size(),
                                   axis),
              "eval_init");
    }
    return {static_cast<void *>(ctx)};
}

/* batch PIR: many tables ("bins") of one entry size behind one context, for keys of one kind
 * (b200dpf_group_create, _et or _xor, named `what` in messages) */
using GroupCreate = std::function<int(b200dpf_ctx **, const int32_t *const *, const int64_t *, int, int, int)>;
std::vector<void *> group_init_with(const std::vector<at::Tensor> &tables, int device, const GroupCreate &create,
                                    const char *what)
{
    TORCH_CHECK(!tables.empty(), what, ": no tables");
    std::vector<at::Tensor> keep;
    std::vector<const int32_t *> ptrs;
    std::vector<int64_t> sizes;
    for (const at::Tensor &t : tables) {
        TORCH_CHECK(t.dim() == 2 && t.size(1) == tables[0].size(1), what, ": tables must be [n_g, entry_size] with one entry_size");
        keep.push_back(t.to(at::kInt).contiguous().cpu());
        ptrs.push_back(keep.back().data_ptr<int32_t>());
        sizes.push_back(keep.back().size(0));
    }
    b200dpf_ctx *ctx = nullptr;
    check(create(&ctx, ptrs.data(), sizes.data(), (int)ptrs.size(), (int)tables[0].size(1), device), what);
    return {static_cast<void *>(ctx)};
}

std::vector<void *> group_init(const std::vector<at::Tensor> &tables, int device)
{
    return group_init_with(tables, device, b200dpf_group_create, "group_init");
}

std::vector<void *> group_init_et(const std::vector<at::Tensor> &tables, int device)
{
    return group_init_with(tables, device, b200dpf_group_create_et, "group_init_et");
}

std::vector<void *> group_init_xor(const std::vector<at::Tensor> &tables, int device)
{
    return group_init_with(tables, device, b200dpf_group_create_xor, "group_init_xor");
}

/* trimmed tables of any row count, for keys of `kind` (B200DPF_KIND_*): b200dpf_create_trimmed and
 * b200dpf_group_create_trimmed; row r is reached by a key for trimmed_alpha(r, n, kind) over trimmed_domain(n, kind) */
Ctx eval_init_trimmed(const at::Tensor &table, int device, int kind)
{
    TORCH_CHECK(table.dim() == 2, "eval_init_trimmed: table must be [num_entries, entry_size]");
    at::Tensor t = table.to(at::kInt).contiguous();
    b200dpf_ctx *ctx = nullptr;
    check(b200dpf_create_trimmed(&ctx, t.data_ptr<int32_t>(), t.size(0), (int)t.size(1), device, kind), "eval_init_trimmed");
    return {static_cast<void *>(ctx)};
}

std::vector<void *> group_init_trimmed(const std::vector<at::Tensor> &tables, int device, int kind)
{
    return group_init_with(
        tables, device,
        [kind](b200dpf_ctx **c, const int32_t *const *t, const int64_t *n, int nbins, int e, int d) {
            return b200dpf_group_create_trimmed(c, t, n, nbins, e, d, kind);
        },
        "group_init_trimmed");
}

int64_t trimmed_domain(int64_t n, int kind)
{
    const int64_t v = b200dpf_trimmed_domain(n, kind);
    TORCH_CHECK(v >= 0, "trimmed_domain: n=", n, " outside [1, 2^31] or unknown kind ", kind);
    return v;
}

int64_t trimmed_alpha(int64_t row, int64_t n, int kind)
{
    const int64_t v = b200dpf_trimmed_alpha(row, n, kind);
    TORCH_CHECK(v >= 0, "trimmed_alpha: row ", row, " of n=", n, " out of range, or unknown kind ", kind);
    return v;
}

/* keys int32 [B,524], bins int32/int64 [B] -> int32 [B, E]: key b evaluated on table bins[b] */
at::Tensor group_eval(const at::Tensor &keys, const at::Tensor &bins, const std::vector<void *> &buffers, int prf)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    TORCH_CHECK(keys.device().is_cpu() && keys.scalar_type() == at::kInt && keys.dim() == 2 && keys.size(1) == kKeyWords &&
                    keys.is_contiguous(),
                "group_eval: keys must be a contiguous CPU int32 tensor [B, 524]");
    at::Tensor b32 = bins.to(at::kInt).contiguous().cpu();
    TORCH_CHECK(b32.dim() == 1 && b32.size(0) == keys.size(0), "group_eval: one bin index per key");
    at::Tensor result = torch::empty({keys.size(0), (int64_t)b200dpf_ctx_entry_size(ctx)}, at::kInt);
    {
        py::gil_scoped_release nogil;
        check(b200dpf_group_eval(ctx, keys.data_ptr<int32_t>(), b32.data_ptr<int32_t>(), keys.size(0), prf,
                                 result.data_ptr<int32_t>()),
              "group_eval");
    }
    return result;
}

/* the same from device keys (int32 [nkeys, 524] at keys_ptr) into device results (int32 [nkeys, E] at out_ptr),
 * enqueued on the stream handle passed as an integer; bins is a CPU int32 tensor [nkeys] (the launch is planned
 * from it on the host) */
void group_eval_device(int64_t keys_ptr, const at::Tensor &bins, int64_t nkeys, const std::vector<void *> &buffers, int prf,
                       int64_t out_ptr, int64_t stream)
{
    TORCH_CHECK(bins.device().is_cpu(), "group_eval_device: bins must be a CPU tensor (the host plans the launch from "
                "them, and reading them from the device would need a synchronisation)");
    TORCH_CHECK(bins.scalar_type() == at::kInt && bins.dim() == 1 && bins.is_contiguous() && bins.size(0) == nkeys,
                "group_eval_device: bins must be a contiguous CPU int32 tensor [nkeys]");
    check(b200dpf_group_eval_device(ctx_of(buffers), reinterpret_cast<const void *>(keys_ptr), bins.data_ptr<int32_t>(), nkeys,
                                    prf, reinterpret_cast<void *>(out_ptr), reinterpret_cast<void *>(stream)),
          "group_eval_device");
}

/* the same with the bins in device memory too (b200dpf_group_eval_device_bins): int32 [nkeys] at bins_ptr, planned on
 * the GPU; a key whose bin is out of range gets a zero row, and their number goes to the int64 at bad_ptr if it is not
 * 0.  Enqueued on the stream handle passed as an integer, with no host wait. */
void group_eval_device_bins(int64_t keys_ptr, int64_t bins_ptr, int64_t nkeys, const std::vector<void *> &buffers, int prf,
                            int64_t out_ptr, int64_t bad_ptr, int64_t stream)
{
    check(b200dpf_group_eval_device_bins(ctx_of(buffers), reinterpret_cast<const void *>(keys_ptr),
                                         reinterpret_cast<const int32_t *>(bins_ptr), nkeys, prf, reinterpret_cast<void *>(out_ptr),
                                         reinterpret_cast<int64_t *>(bad_ptr), reinterpret_cast<void *>(stream)),
          "group_eval_device_bins");
}

/* batch-PIR queries of one key per bin (b200dpf_group_eval_queries_device): device keys at keys_ptr, int32
 * [nqueries, nbins, 524], or with `compact` uint8 [nqueries, group_query_bytes] compact queries, into device
 * results int32 [nqueries, nbins, E] at out_ptr, enqueued on the stream handle passed as an integer */
void group_eval_queries_device(int64_t keys_ptr, int64_t nqueries, const std::vector<void *> &buffers, int prf, int64_t out_ptr,
                               int64_t stream, bool compact)
{
    check(b200dpf_group_eval_queries_device(ctx_of(buffers), reinterpret_cast<const void *>(keys_ptr),
                                            compact ? B200DPF_KEYS_COMPACT : B200DPF_KEYS_WIRE, nqueries, prf,
                                            reinterpret_cast<void *>(out_ptr), reinterpret_cast<void *>(stream)),
          "group_eval_queries_device");
}

/* both servers' batch-PIR queries made on the GPU (b200dpf_group_gen_queries_device): alphas int64 [nqueries, nbins]
 * at alphas_ptr, seeds uint8 [nqueries, nbins, 44] at seeds_ptr, into int32 [nqueries, nbins, 524] wire-format keys
 * or with `compact` uint8 [nqueries, group_query_bytes] compact queries at out_a_ptr and out_b_ptr, enqueued on the
 * stream handle passed as an integer */
void group_gen_queries_device(int64_t alphas_ptr, int64_t seeds_ptr, int64_t nqueries, const std::vector<void *> &buffers,
                              int prf, int64_t out_a_ptr, int64_t out_b_ptr, int64_t stream, bool compact)
{
    check(b200dpf_group_gen_queries_device(ctx_of(buffers), reinterpret_cast<const int64_t *>(alphas_ptr),
                                           reinterpret_cast<const uint8_t *>(seeds_ptr), nqueries, prf,
                                           compact ? B200DPF_KEYS_COMPACT : B200DPF_KEYS_WIRE, reinterpret_cast<void *>(out_a_ptr),
                                           reinterpret_cast<void *>(out_b_ptr), reinterpret_cast<void *>(stream)),
          "group_gen_queries_device");
}

/* row updates of a live table (b200dpf_update_rows): indices int64 [count] natural, rows int32 [count, E],
 * both CPU tensors; synchronous */
void update_rows(const at::Tensor &indices, const at::Tensor &rows, const std::vector<void *> &buffers)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    TORCH_CHECK(indices.device().is_cpu() && indices.scalar_type() == at::kLong && indices.dim() == 1 && indices.is_contiguous(),
                "update_rows: indices must be a contiguous CPU int64 tensor [count]");
    TORCH_CHECK(rows.device().is_cpu() && rows.scalar_type() == at::kInt && rows.dim() == 2 && rows.is_contiguous() &&
                    rows.size(0) == indices.size(0) && rows.size(1) == b200dpf_ctx_entry_size(ctx),
                "update_rows: rows must be a contiguous CPU int32 tensor [count, entry_size]");
    py::gil_scoped_release nogil;
    check(b200dpf_update_rows(ctx, indices.data_ptr<int64_t>(), rows.data_ptr<int32_t>(), indices.size(0)), "update_rows");
}

/* the same from device buffers, enqueued on the stream handle passed as an integer */
void update_rows_device(int64_t idx_ptr, int64_t rows_ptr, int64_t count, const std::vector<void *> &buffers, int64_t stream)
{
    check(b200dpf_update_rows_device(ctx_of(buffers), reinterpret_cast<const int64_t *>(idx_ptr),
                                     reinterpret_cast<const int32_t *>(rows_ptr), count, reinterpret_cast<void *>(stream)),
          "update_rows_device");
}

/* grouped context: row indices[j] of bin bins[j] := rows[j]; CPU tensors, synchronous */
void group_update_rows(const at::Tensor &bins, const at::Tensor &indices, const at::Tensor &rows, const std::vector<void *> &buffers)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    TORCH_CHECK(bins.device().is_cpu() && bins.scalar_type() == at::kInt && bins.dim() == 1 && bins.is_contiguous(),
                "group_update_rows: bins must be a contiguous CPU int32 tensor [count]");
    TORCH_CHECK(indices.device().is_cpu() && indices.scalar_type() == at::kLong && indices.sizes() == bins.sizes() &&
                    indices.is_contiguous(),
                "group_update_rows: indices must be a contiguous CPU int64 tensor [count]");
    TORCH_CHECK(rows.device().is_cpu() && rows.scalar_type() == at::kInt && rows.dim() == 2 && rows.is_contiguous() &&
                    rows.size(0) == indices.size(0) && rows.size(1) == b200dpf_ctx_entry_size(ctx),
                "group_update_rows: rows must be a contiguous CPU int32 tensor [count, entry_size]");
    py::gil_scoped_release nogil;
    check(b200dpf_group_update_rows(ctx, bins.data_ptr<int32_t>(), indices.data_ptr<int64_t>(), rows.data_ptr<int32_t>(),
                                    indices.size(0)),
          "group_update_rows");
}

/* batch codes (b200dpf_batchcode_*): one table [n, E] (CPU or CUDA tensor) in nbins bins of three copies per row */
std::vector<void *> batchcode_init(const at::Tensor &table, int nbins, uint64_t seed, int device, int kind)
{
    TORCH_CHECK(table.dim() == 2, "batchcode_init: table must be [num_entries, entry_size]");
    at::Tensor t = table.to(at::kInt).contiguous();
    b200dpf_ctx *ctx = nullptr;
    {
        py::gil_scoped_release nogil;
        check(b200dpf_batchcode_create(&ctx, t.data_ptr<int32_t>(), t.size(0), (int)t.size(1), nbins, seed, device, kind),
              "batchcode_init");
    }
    return {static_cast<void *>(ctx)};
}

/* (n, nbins, layout seed) of a batch-code context */
py::tuple batchcode_layout(const std::vector<void *> &buffers)
{
    int64_t n = 0;
    int nbins = 0;
    uint64_t seed = 0;
    check(b200dpf_batchcode_layout(ctx_of(buffers), &n, &nbins, &seed), "batchcode_layout");
    return py::make_tuple(n, nbins, seed);
}

/* ([bin of copy c], [in-bin row of copy c]) for c = 0, 1, 2 */
py::tuple batchcode_locate(int64_t n, int nbins, uint64_t seed, int64_t row)
{
    int32_t bins[3];
    int64_t rows[3];
    check(b200dpf_batchcode_locate(n, nbins, seed, row, bins, rows), "batchcode_locate");
    return py::make_tuple(std::vector<int32_t>(bins, bins + 3), std::vector<int64_t>(rows, rows + 3));
}

/* the host plan: wanted int64 [Q, k] CPU tensor -> (alphas int64 [Q, nbins], slots int32 [Q, k]) */
std::vector<at::Tensor> batchcode_plan(int64_t n, int nbins, uint64_t seed, const at::Tensor &wanted)
{
    TORCH_CHECK(wanted.device().is_cpu() && wanted.scalar_type() == at::kLong && wanted.dim() == 2 && wanted.is_contiguous(),
                "batchcode_plan: wanted must be a contiguous CPU int64 tensor [Q, k]");
    at::Tensor alphas = torch::empty({wanted.size(0), (int64_t)std::max(nbins, 0)}, at::kLong);
    at::Tensor slots = torch::empty({wanted.size(0), wanted.size(1)}, at::kInt);
    {
        py::gil_scoped_release nogil;
        check(b200dpf_batchcode_plan(n, nbins, seed, wanted.data_ptr<int64_t>(), wanted.size(0), (int)wanted.size(1),
                                     alphas.data_ptr<int64_t>(), slots.data_ptr<int32_t>()),
              "batchcode_plan");
    }
    return {alphas, slots};
}

/* the device plan (b200dpf_batchcode_plan_device): wanted int64 [nqueries, k] at wanted_ptr, into alphas int64
 * [nqueries, nbins] at alphas_ptr and slots int32 [nqueries, k] at slots_ptr, enqueued on the stream handle passed as
 * an integer */
void batchcode_plan_device(int64_t wanted_ptr, int64_t nqueries, int k, const std::vector<void *> &buffers, int64_t alphas_ptr,
                           int64_t slots_ptr, int64_t stream)
{
    check(b200dpf_batchcode_plan_device(ctx_of(buffers), reinterpret_cast<const int64_t *>(wanted_ptr), nqueries, k,
                                        reinterpret_cast<int64_t *>(alphas_ptr), reinterpret_cast<int32_t *>(slots_ptr),
                                        reinterpret_cast<void *>(stream)),
          "batchcode_plan_device");
}

/* table row indices[j] := rows[j] in all three copies; CPU tensors, synchronous */
void batchcode_update_rows(const at::Tensor &indices, const at::Tensor &rows, const std::vector<void *> &buffers)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    TORCH_CHECK(indices.device().is_cpu() && indices.scalar_type() == at::kLong && indices.dim() == 1 && indices.is_contiguous(),
                "batchcode_update_rows: indices must be a contiguous CPU int64 tensor [count]");
    TORCH_CHECK(rows.device().is_cpu() && rows.scalar_type() == at::kInt && rows.dim() == 2 && rows.is_contiguous() &&
                    rows.size(0) == indices.size(0) && rows.size(1) == b200dpf_ctx_entry_size(ctx),
                "batchcode_update_rows: rows must be a contiguous CPU int32 tensor [count, entry_size]");
    py::gil_scoped_release nogil;
    check(b200dpf_batchcode_update_rows(ctx, indices.data_ptr<int64_t>(), rows.data_ptr<int32_t>(), indices.size(0)),
          "batchcode_update_rows");
}

/* keyword PIR (b200dpf_kwpir_*): keywords int64 [n] (the uint64 keywords' bits) and values [n, E], CPU or CUDA tensors.
 * An empty buffer list when the placement does not finish (B200DPF_EFULL), so the caller can retry another seed; any
 * other failure raises. */
std::vector<void *> kwpir_init(const at::Tensor &keywords, const at::Tensor &values, int64_t m, uint64_t seed, int device, int kind)
{
    TORCH_CHECK(keywords.dim() == 1 && keywords.scalar_type() == at::kLong, "kwpir_init: keywords must be an int64 tensor [n]");
    TORCH_CHECK(values.dim() == 2 && values.size(0) == keywords.size(0), "kwpir_init: values must be [n, value_size]");
    at::Tensor k = keywords.contiguous();
    at::Tensor v = values.to(at::kInt).contiguous();
    b200dpf_ctx *ctx = nullptr;
    int rc;
    {
        py::gil_scoped_release nogil;
        rc = b200dpf_kwpir_create(&ctx, reinterpret_cast<const uint64_t *>(k.data_ptr<int64_t>()), v.data_ptr<int32_t>(), k.size(0),
                                  (int)v.size(1), m, seed, device, kind);
    }
    if (rc == B200DPF_EFULL) return {};
    check(rc, "kwpir_init");
    return {static_cast<void *>(ctx)};
}

/* (n, m, layout seed, value size) of a keyword-PIR context */
py::tuple kwpir_layout(const std::vector<void *> &buffers)
{
    int64_t n = 0, m = 0;
    uint64_t seed = 0;
    int value_size = 0;
    check(b200dpf_kwpir_layout(ctx_of(buffers), &n, &m, &seed, &value_size), "kwpir_layout");
    return py::make_tuple(n, m, seed, value_size);
}

/* (rounds, placement device ms) of a keyword-PIR context's build */
py::tuple kwpir_build_stats(const std::vector<void *> &buffers)
{
    int rounds = 0;
    double ms = 0;
    check(b200dpf_kwpir_build_stats(ctx_of(buffers), &rounds, &ms), "kwpir_build_stats");
    return py::make_tuple(rounds, ms);
}

/* the host locator: keywords int64 [Q] CPU tensor -> rows int64 [Q, 3] */
at::Tensor kwpir_locate(int64_t m, uint64_t seed, const at::Tensor &keywords)
{
    TORCH_CHECK(keywords.device().is_cpu() && keywords.scalar_type() == at::kLong && keywords.dim() == 1 && keywords.is_contiguous(),
                "kwpir_locate: keywords must be a contiguous CPU int64 tensor [Q]");
    at::Tensor rows = torch::empty({keywords.size(0), 3}, at::kLong);
    check(b200dpf_kwpir_locate(m, seed, reinterpret_cast<const uint64_t *>(keywords.data_ptr<int64_t>()), keywords.size(0),
                               rows.data_ptr<int64_t>()),
          "kwpir_locate");
    return rows;
}

/* the device locator (b200dpf_kwpir_plan_device): keywords [nqueries] at keywords_ptr into alphas int64 [nqueries, 3] at
 * alphas_ptr, enqueued on the stream handle passed as an integer */
void kwpir_plan_device(int64_t keywords_ptr, int64_t nqueries, const std::vector<void *> &buffers, int64_t alphas_ptr, int64_t stream)
{
    check(b200dpf_kwpir_plan_device(ctx_of(buffers), reinterpret_cast<const uint64_t *>(keywords_ptr), nqueries,
                                    reinterpret_cast<int64_t *>(alphas_ptr), reinterpret_cast<void *>(stream)),
          "kwpir_plan_device");
}

/* the value of keywords[j] := values[j]; CPU tensors, synchronous */
void kwpir_update(const at::Tensor &keywords, const at::Tensor &values, const std::vector<void *> &buffers)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    TORCH_CHECK(keywords.device().is_cpu() && keywords.scalar_type() == at::kLong && keywords.dim() == 1 && keywords.is_contiguous(),
                "kwpir_update: keywords must be a contiguous CPU int64 tensor [count]");
    TORCH_CHECK(values.device().is_cpu() && values.scalar_type() == at::kInt && values.dim() == 2 && values.is_contiguous() &&
                    values.size(0) == keywords.size(0) && values.size(1) == b200dpf_ctx_entry_size(ctx) - 2,
                "kwpir_update: values must be a contiguous CPU int32 tensor [count, value_size]");
    py::gil_scoped_release nogil;
    check(b200dpf_kwpir_update(ctx, reinterpret_cast<const uint64_t *>(keywords.data_ptr<int64_t>()), values.data_ptr<int32_t>(),
                               keywords.size(0)),
          "kwpir_update");
}

/* every slot's stored tag, int64 [3, m] (the uint64 tags' bits; 0 = empty) */
at::Tensor kwpir_tags(const std::vector<void *> &buffers)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    int64_t n = 0, m = 0;
    uint64_t seed = 0;
    int value_size = 0;
    check(b200dpf_kwpir_layout(ctx, &n, &m, &seed, &value_size), "kwpir_tags");
    at::Tensor tags = torch::empty({3, m}, at::kLong);
    check(b200dpf_kwpir_tags(ctx, reinterpret_cast<uint64_t *>(tags.data_ptr<int64_t>())), "kwpir_tags");
    return tags;
}

/* "all" / "" -> every visible device; "0,2,3" -> that list */
std::vector<int> parse_devices(const std::string &spec)
{
    std::vector<int> devs;
    if (spec.empty() || spec == "all") {
        const int n = (int)at::detail::getCUDAHooks().deviceCount();
        for (int i = 0; i < n; i++) devs.push_back(i);
        return devs;
    }
    size_t pos = 0;
    while (pos < spec.size()) {
        size_t next = spec.find(',', pos);
        if (next == std::string::npos) next = spec.size();
        devs.push_back(std::stoi(spec.substr(pos, next - pos)));
        pos = next + 1;
    }
    return devs;
}

/* dpf_wrapper.cu:93-132.  The reference's eval_init has no device argument (device 0, implicitly);
 * B200DPF_DEVICES=all|0,1,.. in the environment makes this same call spread the table over several
 * GPUs, so the reference's unmodified dpf.py / benchmark.py scale without a launcher. */
std::vector<void *> eval_init(const at::Tensor &table)
{
    const char *env = std::getenv("B200DPF_DEVICES");
    if (env && *env) {
        std::vector<int> devs = parse_devices(env);
        if (devs.size() > 1) {
            const char *ax = std::getenv("B200DPF_AXIS");
            const std::string a = ax ? ax : "auto";
            return eval_init_multi(table, devs, a == "entries" ? B200DPF_AXIS_ENTRIES : (a == "keys" ? B200DPF_AXIS_KEYS : B200DPF_AXIS_AUTO));
        }
        if (devs.size() == 1) return eval_init_sharded(table, devs[0], 0, 1);
    }
    return eval_init_sharded(table, 0, 0, 1);
}

/* dpf_wrapper.cu:86-91 */
void eval_free(const std::vector<void *> &buffers)
{
    if (!buffers.empty() && buffers[0]) b200dpf_destroy(static_cast<b200dpf_ctx *>(buffers[0]));
}

/* keys as one int32[B,524] CPU tensor -> int32[B,E] CPU tensor */
at::Tensor eval_gpu_packed(const at::Tensor &keys, const std::vector<void *> &buffers, int prf)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    TORCH_CHECK(keys.device().is_cpu() && keys.scalar_type() == at::kInt && keys.dim() == 2 &&
                    keys.size(1) == kKeyWords && keys.is_contiguous(),
                "eval_gpu_packed: keys must be a contiguous CPU int32 tensor [B, 524]");
    const int64_t nkeys = keys.size(0);
    at::Tensor result = torch::empty({nkeys, (int64_t)b200dpf_ctx_entry_size(ctx)}, at::kInt);
    {
        py::gil_scoped_release nogil;
        check(b200dpf_eval(ctx, keys.data_ptr<int32_t>(), nkeys, prf, result.data_ptr<int32_t>()), "eval_gpu");
    }
    return result;
}

/* keys in the compact wire form (key_pack), concatenated: uint8 CPU tensor [B * packed_size] or
 * [B, packed_size] -> int32[B,E] CPU tensor.  The buffer is copied to the device as it is. */
at::Tensor eval_gpu_compact(const at::Tensor &packed, int64_t nkeys, const std::vector<void *> &buffers, int prf)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    TORCH_CHECK(packed.device().is_cpu() && packed.scalar_type() == at::kByte && packed.is_contiguous(),
                "eval_gpu_compact: packed keys must be a contiguous CPU uint8 tensor");
    /* the keys' n: the table's rows, or on a trimmed context trimmed_domain(rows) for the context's kind */
    const int per_leaf = b200dpf_ctx_rows_per_leaf(ctx);
    int64_t n = b200dpf_ctx_n(ctx);
    if (b200dpf_ctx_trimmed(ctx) == 1)
        n = b200dpf_trimmed_domain(n, per_leaf == 1 ? B200DPF_KIND_STANDARD : per_leaf == 4 ? B200DPF_KIND_ET : B200DPF_KIND_XOR);
    int depth = 0;   /* of the tree: over leaves, which are rows_per_leaf rows each */
    for (n /= per_leaf; n > 1; n >>= 1) depth++;
    TORCH_CHECK(nkeys >= 1 && (int64_t)packed.numel() == nkeys * (int64_t)b200dpf_key_packed_size(depth),
                "eval_gpu_compact: expected ", nkeys, " keys of ", b200dpf_key_packed_size(depth), " bytes");
    at::Tensor result = torch::empty({nkeys, (int64_t)b200dpf_ctx_entry_size(ctx)}, at::kInt);
    {
        py::gil_scoped_release nogil;
        check(b200dpf_eval_packed(ctx, packed.data_ptr<uint8_t>(), nkeys, prf, result.data_ptr<int32_t>()), "eval_gpu");
    }
    return result;
}

/* Data pointers of a Python list of int32[524] CPU key tensors, without building a
 * std::vector<at::Tensor> (512 reference-count round trips per call): the list is walked with the
 * CPython API and each element unwrapped in place.  `unique` = length with trailing repeats of the
 * SAME tensor object dropped (the reference's dpf.py pads short batches that way, dpf.py:126). */
std::vector<const int32_t *> key_pointers(const py::object &keys_in, int64_t *unique)
{
    /* any sequence is accepted; a list (what dpf.py passes) is walked in place */
    const py::list keys = py::isinstance<py::list>(keys_in) ? py::reinterpret_borrow<py::list>(keys_in) : py::list(keys_in);
    const int64_t total = (int64_t)PyList_GET_SIZE(keys.ptr());
    std::vector<const int32_t *> ptrs((size_t)total);
    PyObject *prev = nullptr;
    int64_t uniq = 0;
    for (int64_t i = 0; i < total; i++) {
        PyObject *o = PyList_GET_ITEM(keys.ptr(), i);
        if (o == prev) {                         /* same object as its predecessor: same pointer */
            ptrs[(size_t)i] = ptrs[(size_t)i - 1];
            continue;
        }
        TORCH_CHECK(THPVariable_Check(o), "dpf_cpp: keys must be torch tensors");
        ptrs[(size_t)i] = key_ptr(THPVariable_Unpack(o));
        prev = o;
        uniq = i + 1;
    }
    if (unique) *unique = uniq;
    return ptrs;
}

/* keys as a Python list of int32[524] CPU tensors, any length -> int32[len, E] CPU tensor */
at::Tensor eval_gpu_list(const py::object &keys, const std::vector<void *> &buffers, int prf)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    int64_t unique = 0;
    std::vector<const int32_t *> ptrs = key_pointers(keys, &unique);
    const int64_t total = (int64_t)ptrs.size();
    at::Tensor result = torch::empty({total, (int64_t)b200dpf_ctx_entry_size(ctx)}, at::kInt);
    if (total == 0) return result;
    {
        py::gil_scoped_release nogil;
        check(b200dpf_eval_gather(ctx, ptrs.data(), total, prf, result.data_ptr<int32_t>()), "eval_gpu");
    }
    return result;
}

/* dpf_wrapper.cu:134-186.  The reference's dpf.py pads short batches by repeating the LAST key
 * object (dpf.py:126); trailing repeats of one tensor are evaluated once and their rows replicated. */
at::Tensor eval_gpu(const py::object &keys, const std::vector<void *> &buffers, int64_t n, int prf)
{
    b200dpf_ctx *ctx = ctx_of(buffers);
    TORCH_CHECK(n == b200dpf_ctx_n(ctx), "eval_gpu: n does not match the initialised table");
    int64_t unique = 0;
    std::vector<const int32_t *> ptrs = key_pointers(keys, &unique);
    TORCH_CHECK(!ptrs.empty(), "eval_gpu: no keys");
    const int64_t total = (int64_t)ptrs.size();
    const int64_t esz = b200dpf_ctx_entry_size(ctx);
    at::Tensor result = torch::empty({total, esz}, at::kInt);
    int32_t *r = result.data_ptr<int32_t>();
    {
        py::gil_scoped_release nogil;
        check(b200dpf_eval_gather(ctx, ptrs.data(), unique, prf, r), "eval_gpu");
    }
    for (int64_t i = unique; i < total; i++) std::memcpy(r + i * esz, r + (unique - 1) * esz, sizeof(int32_t) * (size_t)esz);
    return result;
}

/* device-resident evaluation on the current torch stream handle passed as an integer */
void eval_gpu_device(int64_t keys_ptr, int64_t nkeys, const std::vector<void *> &buffers, int prf, int64_t out_ptr,
                     int64_t stream, bool accumulate)
{
    auto fn = accumulate ? b200dpf_eval_device_acc : b200dpf_eval_device;
    check(fn(ctx_of(buffers), reinterpret_cast<const void *>(keys_ptr), nkeys, prf, reinterpret_cast<void *>(out_ptr),
             reinterpret_cast<void *>(stream)),
          "eval_gpu_device");
}

void expand_gpu_device(int64_t keys_ptr, int64_t nkeys, const std::vector<void *> &buffers, int prf, int64_t out_ptr,
                       int64_t stream)
{
    check(b200dpf_expand_device(ctx_of(buffers), reinterpret_cast<const void *>(keys_ptr), nkeys, prf,
                                reinterpret_cast<void *>(out_ptr), reinterpret_cast<void *>(stream)),
          "expand_gpu_device");
}

int last_launches(const std::vector<void *> &buffers) { return b200dpf_ctx_last_launches(ctx_of(buffers)); }

void set_subtree_log2(const std::vector<void *> &buffers, int s)
{
    check(b200dpf_ctx_set_subtree_log2(ctx_of(buffers), s), "set_subtree_log2");
}

void set_option(const std::vector<void *> &buffers, const std::string &name, int value)
{
    check(b200dpf_ctx_set_option(ctx_of(buffers), name.c_str(), value), "set_option");
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m)
{
    /* the reference surface, dpf_wrapper.cu:190-203 */
    m.def("gen", &gen, "dpf gen");
    m.def("eval_cpu", &eval_cpu, "dpf eval cpu");
    m.def("eval_gpu", &eval_gpu, "dpf eval gpu");
    m.def("eval_init", &eval_init, "dpf eval init");
    m.def("eval_free", &eval_free, "dpf eval free");

    m.attr("ENTRY_SIZE") = py::int_(B200DPF_DEFAULT_ENTRY_SIZE);
    m.attr("BATCH_SIZE") = py::int_(B200DPF_DEFAULT_BATCH_SIZE);
    m.attr("PRF_DUMMY") = py::int_((int)B200DPF_PRF_DUMMY);
    m.attr("PRF_SALSA20") = py::int_((int)B200DPF_PRF_SALSA20);
    m.attr("PRF_CHACHA20") = py::int_((int)B200DPF_PRF_CHACHA20);
    m.attr("PRF_AES128") = py::int_((int)B200DPF_PRF_AES128);

    /* additions */
    m.attr("NATIVE_SHAPES") = py::int_(1);
    m.def("version", []() { return std::string(b200dpf_version()); });
    m.def("key_pack", &key_pack, "compact wire form of a key (bytes)");
    m.def("key_unpack", &key_unpack, "restore an int32[524] key from its compact form");
    m.def("gen_secure", &gen_secure, "dpf gen from a ChaCha20 DRBG (seed: >= 44 bytes)");
    m.def("gen_batch_secure", &gen_batch_secure, "batched keygen from a ChaCha20 DRBG (44 seed bytes per key)", py::arg("alphas"),
          py::arg("n"), py::arg("seeds"), py::arg("prf"), py::arg("nthreads") = 0);
    m.def("gen_batch", &gen_batch, "batched multi-threaded keygen", py::arg("alphas"), py::arg("n"), py::arg("seeds"),
          py::arg("prf"), py::arg("nthreads") = 0);
    m.def("eval_init_sharded", &eval_init_sharded, "eval_init for one entry-range shard", py::arg("table"),
          py::arg("device"), py::arg("shard_rank"), py::arg("shard_count"));
    m.def("group_init", &group_init, "batch PIR: one context over many tables (bins)", py::arg("tables"), py::arg("device") = 0);
    m.def("group_init_et", &group_init_et, "batch PIR for early-terminated keys (four rows per leaf)", py::arg("tables"),
          py::arg("device") = 0);
    m.def("group_init_xor", &group_init_xor, "batch PIR for XOR-shared keys (128 rows per leaf, XOR results)",
          py::arg("tables"), py::arg("device") = 0);
    m.def("eval_init_trimmed", &eval_init_trimmed, "eval_init for a table of any row count (trimmed context)",
          py::arg("table"), py::arg("device") = 0, py::arg("kind") = 0);
    m.def("group_init_trimmed", &group_init_trimmed, "batch PIR over bins of any row count (trimmed context)",
          py::arg("tables"), py::arg("device") = 0, py::arg("kind") = 0);
    m.def("trimmed_domain", &trimmed_domain, "n of the keys a trimmed table of n rows takes", py::arg("n"), py::arg("kind") = 0);
    m.def("trimmed_alpha", &trimmed_alpha, "key index of row `row` of a trimmed n-row table", py::arg("row"), py::arg("n"),
          py::arg("kind") = 0);
    m.def("table_rows", [](const std::vector<void *> &b) { return b200dpf_ctx_table_rows(ctx_of(b)); },
          "rows of the context's device table, padding included");
    m.def("group_eval", &group_eval, "batch PIR: evaluate (bin, key) pairs in one launch");
    m.def("group_eval_device", &group_eval_device, "batch PIR from device keys into device results, enqueued on a stream",
          py::arg("keys_ptr"), py::arg("bins"), py::arg("nkeys"), py::arg("buffers"), py::arg("prf"), py::arg("out_ptr"),
          py::arg("stream"));
    m.def("group_eval_device_bins", &group_eval_device_bins,
          "batch PIR from device keys and device bins into device results, planned on the GPU, enqueued on a stream",
          py::arg("keys_ptr"), py::arg("bins_ptr"), py::arg("nkeys"), py::arg("buffers"), py::arg("prf"), py::arg("out_ptr"),
          py::arg("bad_ptr"), py::arg("stream"));
    m.def("group_eval_queries_device", &group_eval_queries_device,
          "batch PIR: queries of one key per bin from device memory into device results, enqueued on a stream",
          py::arg("keys_ptr"), py::arg("nqueries"), py::arg("buffers"), py::arg("prf"), py::arg("out_ptr"), py::arg("stream"),
          py::arg("compact") = false);
    m.def("group_gen_queries_device", &group_gen_queries_device,
          "batch PIR: both servers' queries of one key per bin made on the GPU from device rows and seeds, enqueued on a stream",
          py::arg("alphas_ptr"), py::arg("seeds_ptr"), py::arg("nqueries"), py::arg("buffers"), py::arg("prf"),
          py::arg("out_a_ptr"), py::arg("out_b_ptr"), py::arg("stream"), py::arg("compact") = false);
    m.def("group_query_bytes", [](const std::vector<void *> &b) { return b200dpf_group_query_bytes(ctx_of(b)); },
          "bytes of one compact query of a grouped context (one compact key per bin); -1 if not grouped");
    m.def("eval_init_multi", &eval_init_multi, "eval_init over several GPUs of this process", py::arg("table"),
          py::arg("devices"), py::arg("axis") = 0);
    m.def("update_rows", &update_rows, "table[indices[j]] := rows[j] on a live context (CPU tensors)");
    m.def("update_rows_device", &update_rows_device, "row update from device buffers, enqueued on a stream",
          py::arg("idx_ptr"), py::arg("rows_ptr"), py::arg("count"), py::arg("buffers"), py::arg("stream"));
    m.def("group_update_rows", &group_update_rows, "batch PIR: row indices[j] of bin bins[j] := rows[j]");
    m.def("batchcode_init", &batchcode_init, "batch code: one table in nbins bins, three copies per row", py::arg("table"),
          py::arg("nbins"), py::arg("seed"), py::arg("device") = 0, py::arg("kind") = 0);
    m.def("batchcode_layout", &batchcode_layout, "(n, nbins, layout seed) of a batch-code context");
    m.def("batchcode_locate", &batchcode_locate, "(bins, in-bin rows) of the three copies of a row", py::arg("n"),
          py::arg("nbins"), py::arg("seed"), py::arg("row"));
    m.def("batchcode_plan", &batchcode_plan, "the client's plan: wanted [Q, k] -> (alphas [Q, nbins], slots [Q, k])",
          py::arg("n"), py::arg("nbins"), py::arg("seed"), py::arg("wanted"));
    m.def("batchcode_plan_device", &batchcode_plan_device, "the client's plan on the GPU, from and into device buffers",
          py::arg("wanted_ptr"), py::arg("nqueries"), py::arg("k"), py::arg("buffers"), py::arg("alphas_ptr"),
          py::arg("slots_ptr"), py::arg("stream") = 0);
    m.def("batchcode_update_rows", &batchcode_update_rows, "batch code: table row indices[j] := rows[j] in all three copies");
    m.def("kwpir_init", &kwpir_init, "keyword PIR: (keyword, value) items placed in 3 tables of m slots; [] if placement fails",
          py::arg("keywords"), py::arg("values"), py::arg("m"), py::arg("seed"), py::arg("device") = 0, py::arg("kind") = 0);
    m.def("kwpir_layout", &kwpir_layout, "(n, m, layout seed, value size) of a keyword-PIR context");
    m.def("kwpir_build_stats", &kwpir_build_stats, "(rounds, placement device ms) of a keyword-PIR context's build");
    m.def("kwpir_locate", &kwpir_locate, "the in-bin rows [Q, 3] of keywords [Q]", py::arg("m"), py::arg("seed"), py::arg("keywords"));
    m.def("kwpir_plan_device", &kwpir_plan_device, "the in-bin rows on the GPU, from and into device buffers", py::arg("keywords_ptr"),
          py::arg("nqueries"), py::arg("buffers"), py::arg("alphas_ptr"), py::arg("stream") = 0);
    m.def("kwpir_update", &kwpir_update, "keyword PIR: the value of keywords[j] := values[j]");
    m.def("kwpir_tags", &kwpir_tags, "every slot's stored tag [3, m] (keyword + 1, 0 = empty)");
    m.def("parse_devices", &parse_devices, "'all' or '0,1,2' -> device list");
    m.def("device_count", [](const std::vector<void *> &b) { return b200dpf_ctx_device_count(ctx_of(b)); });
    m.def("axis", [](const std::vector<void *> &b) { return b200dpf_ctx_axis(ctx_of(b)); });
    m.def("eval_gpu_packed", &eval_gpu_packed, "eval_gpu with keys as one [B,524] tensor");
    m.def("eval_gpu_list", &eval_gpu_list, "eval_gpu with keys as a list of any length");
    m.def("eval_gpu_device", &eval_gpu_device, "device-resident asynchronous evaluation", py::arg("keys_ptr"),
          py::arg("nkeys"), py::arg("buffers"), py::arg("prf"), py::arg("out_ptr"), py::arg("stream"),
          py::arg("accumulate") = false);
    m.def("expand_gpu_device", &expand_gpu_device, "device-resident share-vector expansion");
    m.def("last_launches", &last_launches);
    m.def("set_subtree_log2", &set_subtree_log2);
    m.def("set_option", &set_option, "tuning knob of a live context (include/b200dpf.h: b200dpf_ctx_set_option)");
    m.def("eval_gpu_compact", &eval_gpu_compact, "eval_gpu with keys in the compact wire form (uint8 tensor)");
    m.def("key_packed_size", [](int depth) { return (int64_t)b200dpf_key_packed_size(depth); });
    m.def("gen_et", &gen_et, "early-terminated key pair for row k of an n-row table (seed: >= 44 bytes)");
    m.def("gen_batch_et", &gen_batch_et, "batched early-terminated keygen (44 seed bytes per key)", py::arg("alphas"),
          py::arg("n"), py::arg("seeds"), py::arg("prf"), py::arg("nthreads") = 0);
    m.def("eval_cpu_et", &eval_cpu_et, "share of every row of an early-terminated key on the CPU");
    m.def("key_pack_et", &key_pack_et, "compact wire form (\"DPE4\") of an early-terminated key");
    m.def("key_unpack_et", &key_unpack_et, "restore an early-terminated int32[524] key from its compact form");
    m.def("eval_init_et", &eval_init_et, "eval_init for early-terminated keys (four rows per leaf)", py::arg("table"),
          py::arg("device") = 0, py::arg("shard_rank") = 0, py::arg("shard_count") = 1);
    m.def("rows_per_leaf", [](const std::vector<void *> &b) { return b200dpf_ctx_rows_per_leaf(ctx_of(b)); });
    m.def("gen_xor", &gen_xor, "XOR-shared key pair for row k of an n-row table (seed: >= 44 bytes)");
    m.def("gen_batch_xor", &gen_batch_xor, "batched XOR-shared keygen (44 seed bytes per key)", py::arg("alphas"),
          py::arg("n"), py::arg("seeds"), py::arg("prf"), py::arg("nthreads") = 0);
    m.def("eval_cpu_xor", &eval_cpu_xor, "share bits of every row of an XOR-shared key on the CPU, packed 32 per int32");
    m.def("key_pack_xor", &key_pack_xor, "compact wire form (\"DPX7\") of an XOR-shared key");
    m.def("key_unpack_xor", &key_unpack_xor, "restore an XOR-shared int32[524] key from its compact form");
    m.def("eval_init_xor", &eval_init_xor, "eval_init for XOR-shared keys (128 rows per leaf, XOR results)", py::arg("table"),
          py::arg("device") = 0, py::arg("shard_rank") = 0, py::arg("shard_count") = 1);
}
