"""ctypes binding of the C ABI in include/b200dpf.h.

This is the binding a non-torch host (or the reference's maintainers, see
INTEGRATION.md) would write: plain pointers and sizes over libb200dpf.so.  The
torch-facing module is `dpf_cpp` (csrc/dpf_cpp_ext.cpp); this one is used by the
parity tests and the benchmark, which want to drive the ABI directly.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200dpf.so")
KEY_WORDS = 524
PRF_DUMMY, PRF_SALSA20, PRF_CHACHA20, PRF_AES128 = 0, 1, 2, 3
PRF_NAMES = {0: "DUMMY", 1: "SALSA20", 2: "CHACHA20", 3: "AES128"}
KEYS_WIRE, KEYS_COMPACT = 0, 1

# every symbol include/b200dpf.h declares
SYMBOLS = [
    "b200dpf_version", "b200dpf_last_error", "b200dpf_gen", "b200dpf_gen_secure", "b200dpf_gen_batch", "b200dpf_gen_batch_secure", "b200dpf_gen_batch_gpu", "b200dpf_eval_cpu",
    "b200dpf_key_packed_size", "b200dpf_key_pack", "b200dpf_key_unpack", "b200dpf_key_n", "b200dpf_key_depth", "b200dpf_create", "b200dpf_destroy", "b200dpf_eval",
    "b200dpf_eval_packed", "b200dpf_eval_gather", "b200dpf_ctx_set_option", "b200dpf_create_multi", "b200dpf_ctx_device_count", "b200dpf_ctx_axis", "b200dpf_ctx_read_timing",
    "b200dpf_group_create", "b200dpf_group_eval", "b200dpf_group_eval_device", "b200dpf_group_bins", "b200dpf_ctx_last_device_ms",
    "b200dpf_update_rows", "b200dpf_update_rows_device", "b200dpf_group_update_rows",
    "b200dpf_host_staging", "b200dpf_eval_device", "b200dpf_eval_device_acc", "b200dpf_expand_device", "b200dpf_ctx_n", "b200dpf_ctx_entry_size",
    "b200dpf_ctx_device", "b200dpf_ctx_last_launches", "b200dpf_ctx_set_subtree_log2",
    "b200dpf_gen_et", "b200dpf_gen_batch_et", "b200dpf_eval_cpu_et", "b200dpf_key_pack_et", "b200dpf_key_unpack_et",
    "b200dpf_create_et", "b200dpf_ctx_rows_per_leaf", "b200dpf_group_create_et",
    "b200dpf_gen_xor", "b200dpf_gen_batch_xor", "b200dpf_eval_cpu_xor", "b200dpf_key_pack_xor", "b200dpf_key_unpack_xor",
    "b200dpf_create_xor", "b200dpf_group_create_xor",
    "b200dpf_group_query_bytes", "b200dpf_group_eval_queries_device",
    "b200dpf_gen_batch_gpu_et", "b200dpf_gen_batch_gpu_xor", "b200dpf_group_gen_queries_device",
    "b200dpf_trimmed_domain", "b200dpf_trimmed_alpha", "b200dpf_create_trimmed", "b200dpf_group_create_trimmed",
    "b200dpf_ctx_trimmed", "b200dpf_ctx_table_rows",
    "b200dpf_group_eval_device_bins", "b200dpf_group_plan_lists",
    "b200dpf_batchcode_create", "b200dpf_batchcode_layout", "b200dpf_batchcode_locate", "b200dpf_batchcode_plan",
    "b200dpf_batchcode_plan_device", "b200dpf_batchcode_update_rows",
    "b200dpf_kwpir_create", "b200dpf_kwpir_layout", "b200dpf_kwpir_build_stats", "b200dpf_kwpir_locate",
    "b200dpf_kwpir_plan_device", "b200dpf_kwpir_update", "b200dpf_kwpir_tags",
]

# The kinds of key, by the suffix of their entry points: log2 table rows per leaf, maximum depth, name.  A key
# is slot 0 = (d, lane_bits, 0, 0), 1 <= d <= max depth, slot 130 = 2^(d + lane_bits) as a u64.
KINDS = {
    "": (0, 32, "standard"),
    "_et": (2, 29, "early-terminated"),
    "_xor": (7, 24, "XOR-shared"),
}
# the kind ids of b200dpf_create_trimmed and b200dpf_group_create_trimmed (B200DPF_KIND_*), by suffix
KIND_IDS = {"": 0, "_et": 1, "_xor": 2}

_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(dtype=np.int64, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
_u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")


class B200DPFError(RuntimeError):
    pass


def load():
    if not os.path.exists(LIB_PATH):
        raise ImportError("libb200dpf.so not built (run `python gpu-dpf_b200/build.py`); there is no fallback")
    L = C.CDLL(LIB_PATH)
    L.b200dpf_version.restype = C.c_char_p
    L.b200dpf_last_error.restype = C.c_char_p
    for kind in KINDS:
        getattr(L, "b200dpf_eval_cpu" + kind).argtypes = [_i32p, C.c_int, _u32p if kind == "_xor" else _i32p]
        getattr(L, "b200dpf_key_pack" + kind).argtypes = [_i32p, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
        getattr(L, "b200dpf_key_unpack" + kind).argtypes = [C.c_char_p, C.c_size_t, _i32p]
        getattr(L, "b200dpf_create" + kind).argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int]
    for gen in ("", "_secure", "_et", "_xor"):
        getattr(L, "b200dpf_gen" + gen).argtypes = [C.c_int64, C.c_int64, C.c_char_p, C.c_size_t, C.c_int, _i32p, _i32p]
    for drbg in ("_secure", "_et", "_xor"):   # the ChaCha20-DRBG generators: 44 seed bytes per key
        getattr(L, "b200dpf_gen_batch" + drbg).argtypes = [_i64p, C.c_char_p, C.c_int64, C.c_int64, C.c_int, C.c_int, _i32p, _i32p]
    L.b200dpf_gen_batch.argtypes = [_i64p, _u32p, C.c_int64, C.c_int64, C.c_int, C.c_int, _i32p, _i32p]
    for kind in KINDS:
        getattr(L, "b200dpf_gen_batch_gpu" + kind).argtypes = [_i64p, C.c_char_p, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                                               C.c_void_p, C.c_void_p]
    L.b200dpf_key_packed_size.argtypes = [C.c_int]
    L.b200dpf_key_packed_size.restype = C.c_size_t
    L.b200dpf_key_n.argtypes = [_i32p]
    L.b200dpf_key_n.restype = C.c_int64
    L.b200dpf_key_depth.argtypes = [_i32p]
    L.b200dpf_create_multi.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int]
    L.b200dpf_ctx_device_count.argtypes = [C.c_void_p]
    L.b200dpf_ctx_axis.argtypes = [C.c_void_p]
    L.b200dpf_group_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), _i64p, C.c_int, C.c_int, C.c_int]
    L.b200dpf_group_eval.argtypes = [C.c_void_p, _i32p, _i32p, C.c_int64, C.c_int, _i32p]
    L.b200dpf_group_eval_device.argtypes = [C.c_void_p, C.c_void_p, _i32p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
    L.b200dpf_group_eval_device_bins.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                                 C.c_void_p]
    L.b200dpf_group_plan_lists.argtypes = [C.c_void_p, C.c_int, _i64p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                           C.c_int64]
    L.b200dpf_group_bins.argtypes = [C.c_void_p]
    L.b200dpf_group_query_bytes.argtypes = [C.c_void_p]
    L.b200dpf_group_query_bytes.restype = C.c_int64
    L.b200dpf_group_eval_queries_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
    L.b200dpf_group_gen_queries_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]
    L.b200dpf_ctx_last_device_ms.argtypes = [C.c_void_p]
    L.b200dpf_ctx_last_device_ms.restype = C.c_double
    L.b200dpf_ctx_read_timing.argtypes = [C.c_void_p, np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS"), C.c_int,
                                          C.POINTER(C.c_int)]
    L.b200dpf_update_rows.argtypes = [C.c_void_p, _i64p, _i32p, C.c_int64]
    L.b200dpf_update_rows_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    L.b200dpf_group_update_rows.argtypes = [C.c_void_p, _i32p, _i64p, _i32p, C.c_int64]
    L.b200dpf_destroy.argtypes = [C.c_void_p]
    L.b200dpf_eval.argtypes = [C.c_void_p, _i32p, C.c_int64, C.c_int, _i32p]
    L.b200dpf_eval_packed.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int, _i32p]
    L.b200dpf_eval_gather.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int64, C.c_int, _i32p]
    L.b200dpf_ctx_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    L.b200dpf_host_staging.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.POINTER(C.c_int32))]
    L.b200dpf_eval_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
    L.b200dpf_eval_device_acc.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
    L.b200dpf_expand_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p]
    L.b200dpf_ctx_n.argtypes = [C.c_void_p]
    L.b200dpf_ctx_n.restype = C.c_int64
    L.b200dpf_ctx_entry_size.argtypes = [C.c_void_p]
    L.b200dpf_ctx_device.argtypes = [C.c_void_p]
    L.b200dpf_ctx_last_launches.argtypes = [C.c_void_p]
    L.b200dpf_ctx_set_subtree_log2.argtypes = [C.c_void_p, C.c_int]
    L.b200dpf_ctx_rows_per_leaf.argtypes = [C.c_void_p]
    for kind in ("_et", "_xor"):
        getattr(L, "b200dpf_group_create" + kind).argtypes = L.b200dpf_group_create.argtypes
    L.b200dpf_trimmed_domain.argtypes = [C.c_int64, C.c_int]
    L.b200dpf_trimmed_domain.restype = C.c_int64
    L.b200dpf_trimmed_alpha.argtypes = [C.c_int64, C.c_int64, C.c_int]
    L.b200dpf_trimmed_alpha.restype = C.c_int64
    L.b200dpf_create_trimmed.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int]
    L.b200dpf_group_create_trimmed.argtypes = L.b200dpf_group_create.argtypes + [C.c_int]
    L.b200dpf_ctx_trimmed.argtypes = [C.c_void_p]
    L.b200dpf_ctx_table_rows.argtypes = [C.c_void_p]
    L.b200dpf_ctx_table_rows.restype = C.c_int64
    L.b200dpf_batchcode_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_int,
                                           C.c_int]
    L.b200dpf_batchcode_layout.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    L.b200dpf_batchcode_locate.argtypes = [C.c_int64, C.c_int, C.c_uint64, C.c_int64, _i32p, _i64p]
    L.b200dpf_batchcode_plan.argtypes = [C.c_int64, C.c_int, C.c_uint64, _i64p, C.c_int64, C.c_int, _i64p, _i32p]
    L.b200dpf_batchcode_plan_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200dpf_batchcode_update_rows.argtypes = [C.c_void_p, _i64p, _i32p, C.c_int64]
    L.b200dpf_kwpir_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_uint64,
                                       C.c_int, C.c_int]
    L.b200dpf_kwpir_layout.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_uint64),
                                       C.POINTER(C.c_int)]
    L.b200dpf_kwpir_build_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_double)]
    L.b200dpf_kwpir_locate.argtypes = [C.c_int64, C.c_uint64, _u64p, C.c_int64, _i64p]
    L.b200dpf_kwpir_plan_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    L.b200dpf_kwpir_update.argtypes = [C.c_void_p, _u64p, _i32p, C.c_int64]
    L.b200dpf_kwpir_tags.argtypes = [C.c_void_p, _u64p]
    return L


_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        _LIB = load()
    return _LIB


def _check(rc, what):
    if rc != 0:
        raise B200DPFError("%s failed (%d): %s" % (what, rc, lib().b200dpf_last_error().decode()))


def gen(alpha, n, seed32, prf):
    a = np.zeros(KEY_WORDS, np.int32)
    b = np.zeros(KEY_WORDS, np.int32)
    seed = int(seed32 & 0xFFFFFFFF).to_bytes(4, "little")
    _check(lib().b200dpf_gen(alpha, n, seed, len(seed), prf, a, b), "b200dpf_gen")
    return a, b


def gen_secure(alpha, n, seed_bytes, prf):
    return _gen_drbg("_secure", alpha, n, seed_bytes, prf)


def gen_batch(alphas, n, seeds32, prf, nthreads=0):
    alphas = np.ascontiguousarray(alphas, np.int64)
    seeds32 = np.ascontiguousarray(np.asarray(seeds32, np.int64) & 0xFFFFFFFF, np.uint32)
    a = np.zeros((len(alphas), KEY_WORDS), np.int32)
    b = np.zeros((len(alphas), KEY_WORDS), np.int32)
    _check(lib().b200dpf_gen_batch(alphas, seeds32, len(alphas), n, prf, nthreads, a, b), "b200dpf_gen_batch")
    return a, b


def gen_batch_secure(alphas, n, seed_bytes, prf, nthreads=0):
    """seed_bytes: 44 bytes of entropy per key, concatenated"""
    alphas = np.ascontiguousarray(alphas, np.int64)
    assert len(seed_bytes) == 44 * len(alphas)
    a = np.zeros((len(alphas), KEY_WORDS), np.int32)
    b = np.zeros((len(alphas), KEY_WORDS), np.int32)
    _check(lib().b200dpf_gen_batch_secure(alphas, bytes(seed_bytes), len(alphas), n, prf, nthreads, a, b), "b200dpf_gen_batch_secure")
    return a, b


def gen_batch_gpu(alphas, n, seed_bytes, prf, device=0, out_ptrs=None):
    """GPU keygen; same keys as gen_batch_secure for the same seeds.  out_ptrs=(ptr_a, ptr_b): device
    addresses to leave the keys at (int32 [count, 524] each) instead of returning host arrays."""
    return _gen_batch_gpu("", alphas, n, seed_bytes, prf, device, out_ptrs)


def _gen_batch_gpu(kind, alphas, n, seed_bytes, prf, device, out_ptrs):
    alphas = np.ascontiguousarray(alphas, np.int64)
    name = "b200dpf_gen_batch_gpu" + kind
    assert len(seed_bytes) == 44 * len(alphas)
    if out_ptrs is not None:
        _check(getattr(lib(), name)(alphas, bytes(seed_bytes), len(alphas), n, prf, device,
                                    C.c_void_p(out_ptrs[0]), C.c_void_p(out_ptrs[1])), name)
        return None
    a = np.zeros((len(alphas), KEY_WORDS), np.int32)
    b = np.zeros((len(alphas), KEY_WORDS), np.int32)
    _check(getattr(lib(), name)(alphas, bytes(seed_bytes), len(alphas), n, prf, device,
                                a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p)), name)
    return a, b


def _key_n(key, kind):
    """rows of a key of `kind` (a KINDS suffix), or -1"""
    lane_bits, max_depth, _ = KINDS[kind]
    d = int(key[0])
    if key[1] != lane_bits or key[2] or key[3] or not 1 <= d <= max_depth:
        return -1
    n = int(np.uint32(key[130 * 4])) | int(np.uint32(key[130 * 4 + 1])) << 32
    return n if n == 1 << (d + lane_bits) and not key[130 * 4 + 2:130 * 4 + 4].any() else -1


def _xor_key_n(key):
    """rows of an XOR-shared key, or -1 (_key_n(key, "_xor") under the name existing callers use)"""
    return _key_n(key, "_xor")


def _gen_drbg(suffix, alpha, n, seed_bytes, prf):
    a = np.zeros(KEY_WORDS, np.int32)
    b = np.zeros(KEY_WORDS, np.int32)
    name = "b200dpf_gen" + suffix
    _check(getattr(lib(), name)(alpha, n, bytes(seed_bytes), len(seed_bytes), prf, a, b), name)
    return a, b


def _gen_batch_drbg(kind, alphas, n, seed_bytes, prf, nthreads):
    alphas = np.ascontiguousarray(alphas, np.int64)
    name = "b200dpf_gen_batch" + kind
    if len(seed_bytes) != 44 * len(alphas):
        raise ValueError("gen_batch%s needs 44 seed bytes per key (%d keys, %d bytes)" % (kind, len(alphas), len(seed_bytes)))
    a = np.zeros((len(alphas), KEY_WORDS), np.int32)
    b = np.zeros((len(alphas), KEY_WORDS), np.int32)
    _check(getattr(lib(), name)(alphas, bytes(seed_bytes), len(alphas), n, prf, nthreads, a, b), name)
    return a, b


def _eval_cpu(kind, key, prf):
    key = np.ascontiguousarray(key, np.int32)
    n = _key_n(key, kind)
    if n < 0:
        raise B200DPFError("not an %s key" % KINDS[kind][2] if kind else "malformed key")
    out = np.zeros(n // 32, np.uint32) if kind == "_xor" else np.zeros(n, np.int32)
    name = "b200dpf_eval_cpu" + kind
    _check(getattr(lib(), name)(key, prf, out), name)
    return out


def _key_pack(kind, key):
    key = np.ascontiguousarray(key, np.int32)
    buf = C.create_string_buffer(lib().b200dpf_key_packed_size(32))
    n = C.c_size_t()
    name = "b200dpf_key_pack" + kind
    _check(getattr(lib(), name)(key, buf, len(buf), C.byref(n)), name)
    return buf.raw[:n.value]


def _key_unpack(kind, packed):
    key = np.zeros(KEY_WORDS, np.int32)
    name = "b200dpf_key_unpack" + kind
    _check(getattr(lib(), name)(bytes(packed), len(packed), key), name)
    return key


def key_pack(key):
    return _key_pack("", key)


def key_unpack(packed):
    return _key_unpack("", packed)


def eval_cpu(key, prf):
    return _eval_cpu("", key, prf)


def gen_et(alpha, n, seed_bytes, prf):
    """early-terminated key pair for row alpha of an n-row table (DESIGN.md section 9); >= 44 seed bytes"""
    return _gen_drbg("_et", alpha, n, seed_bytes, prf)


def gen_batch_et(alphas, n, seed_bytes, prf, nthreads=0):
    """seed_bytes: 44 bytes of entropy per key, concatenated"""
    return _gen_batch_drbg("_et", alphas, n, seed_bytes, prf, nthreads)


def gen_batch_gpu_et(alphas, n, seed_bytes, prf, device=0, out_ptrs=None):
    """gen_batch_et on a GPU: the same keys for the same seeds; out_ptrs as for gen_batch_gpu"""
    return _gen_batch_gpu("_et", alphas, n, seed_bytes, prf, device, out_ptrs)


def eval_cpu_et(key, prf):
    return _eval_cpu("_et", key, prf)


def key_pack_et(key):
    return _key_pack("_et", key)


def key_unpack_et(packed):
    return _key_unpack("_et", packed)


def gen_xor(alpha, n, seed_bytes, prf):
    """XOR-shared key pair for row alpha of an n-row table (DESIGN.md section 10); >= 44 seed bytes"""
    return _gen_drbg("_xor", alpha, n, seed_bytes, prf)


def gen_batch_xor(alphas, n, seed_bytes, prf, nthreads=0):
    """seed_bytes: 44 bytes of entropy per key, concatenated"""
    return _gen_batch_drbg("_xor", alphas, n, seed_bytes, prf, nthreads)


def gen_batch_gpu_xor(alphas, n, seed_bytes, prf, device=0, out_ptrs=None):
    """gen_batch_xor on a GPU: the same keys for the same seeds; out_ptrs as for gen_batch_gpu"""
    return _gen_batch_gpu("_xor", alphas, n, seed_bytes, prf, device, out_ptrs)


def eval_cpu_xor(key, prf):
    """share bits packed, uint32 [n / 32]: row i is bit (i & 31) of word i >> 5"""
    return _eval_cpu("_xor", key, prf)


def key_pack_xor(key):
    return _key_pack("_xor", key)


def key_unpack_xor(packed):
    return _key_unpack("_xor", packed)


def _kind_id(kind):
    if kind in KIND_IDS:
        return KIND_IDS[kind]
    if kind in KIND_IDS.values():
        return kind
    raise ValueError("unknown key kind %r (one of %s or 0, 1, 2)" % (kind, sorted(KIND_IDS)))


def trimmed_domain(n, kind=""):
    """the n of the keys a trimmed table of n rows takes (b200dpf_trimmed_domain); kind: "", "_et", "_xor" or its id"""
    N = lib().b200dpf_trimmed_domain(int(n), _kind_id(kind))
    if N < 0:
        raise ValueError("trimmed_domain: n=%d outside [1, 2^31]" % n)
    return N


def trimmed_alpha(row, n, kind=""):
    """the key index of row `row` of a trimmed table of n rows (b200dpf_trimmed_alpha)"""
    a = lib().b200dpf_trimmed_alpha(int(row), int(n), _kind_id(kind))
    if a < 0:
        raise ValueError("trimmed_alpha: row %d of n=%d out of range" % (row, n))
    return a


class Context:
    """One table (or one entry-range shard of it) resident on one GPU.  early_termination=True makes a
    context for early-terminated keys (b200dpf_create_et): four table rows per tree leaf.  xor=True makes
    one for XOR-shared keys (b200dpf_create_xor): 128 rows per leaf, and results that XOR (not add) to
    the selected row.  trimmed=True makes a trimmed context (b200dpf_create_trimmed) of the kind: any number of
    rows, row r reached by a key for trimmed_alpha(r, n) over trimmed_domain(n) rows, update_rows by row number."""

    def __init__(self, table, device=0, shard_rank=0, shard_count=1, early_termination=False, xor=False, trimmed=False):
        if xor and early_termination:
            raise ValueError("a context takes one kind of key: pass xor=True or early_termination=True, not both")
        table = np.ascontiguousarray(table, np.int32)
        assert table.ndim == 2
        self.n, self.entry_size = table.shape
        self.handle = C.c_void_p()
        self.kind = "_xor" if xor else "_et" if early_termination else ""
        if trimmed:
            if (shard_rank, shard_count) != (0, 1):
                raise ValueError("a trimmed context holds the whole table: no shards")
            _check(lib().b200dpf_create_trimmed(C.byref(self.handle), table.ctypes.data_as(C.c_void_p), self.n,
                                                self.entry_size, device, KIND_IDS[self.kind]), "b200dpf_create_trimmed")
            return
        name = "b200dpf_create" + self.kind
        _check(getattr(lib(), name)(C.byref(self.handle), table.ctypes.data_as(C.c_void_p), self.n, self.entry_size,
                                    device, shard_rank, shard_count), name)

    @classmethod
    def multi(cls, table, devices, axis=0):
        """One table over several GPUs of this process; axis 0 auto, 1 entries, 2 keys."""
        table = np.ascontiguousarray(table, np.int32)
        self = cls.__new__(cls)
        self.n, self.entry_size = table.shape
        self.handle = C.c_void_p()
        devs = (C.c_int * len(devices))(*devices)
        _check(lib().b200dpf_create_multi(C.byref(self.handle), table.ctypes.data_as(C.c_void_p), self.n, self.entry_size,
                                          devs, len(devices), axis), "b200dpf_create_multi")
        return self

    @property
    def device_count(self):
        return lib().b200dpf_ctx_device_count(self.handle)

    @property
    def axis(self):
        return lib().b200dpf_ctx_axis(self.handle)

    @classmethod
    def from_device_ptr(cls, ptr, n, entry_size, device=0, shard_rank=0, shard_count=1):
        self = cls.__new__(cls)
        self.n, self.entry_size = n, entry_size
        self.handle = C.c_void_p()
        _check(lib().b200dpf_create(C.byref(self.handle), C.c_void_p(ptr), n, entry_size, device, shard_rank,
                                    shard_count), "b200dpf_create")
        return self

    def eval(self, keys, prf):
        keys = np.ascontiguousarray(keys, np.int32).reshape(-1, KEY_WORDS)
        out = np.zeros((keys.shape[0], self.entry_size), np.int32)
        _check(lib().b200dpf_eval(self.handle, keys, keys.shape[0], prf, out), "b200dpf_eval")
        return out

    def eval_packed(self, packed, nkeys, prf):
        """keys in the compact wire form (key_pack), concatenated"""
        out = np.zeros((nkeys, self.entry_size), np.int32)
        _check(lib().b200dpf_eval_packed(self.handle, bytes(packed), nkeys, prf, out), "b200dpf_eval_packed")
        return out

    def eval_gather(self, key_list, prf):
        """keys as a list of separate int32[524] arrays (the reference's calling convention)"""
        arrs = [np.ascontiguousarray(k, np.int32) for k in key_list]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        out = np.zeros((len(arrs), self.entry_size), np.int32)
        _check(lib().b200dpf_eval_gather(self.handle, ptrs, len(arrs), prf, out), "b200dpf_eval_gather")
        return out

    def update_rows(self, indices, rows):
        """table[indices[j]] := rows[j] (natural indices, last occurrence wins); synchronous"""
        indices = np.ascontiguousarray(indices, np.int64).reshape(-1)
        rows = np.ascontiguousarray(rows, np.int32).reshape(len(indices), self.entry_size)
        _check(lib().b200dpf_update_rows(self.handle, indices, rows, len(indices)), "b200dpf_update_rows")

    def update_rows_device(self, idx_ptr, rows_ptr, count, stream=0):
        """update_rows from device buffers (int64 [count], int32 [count, entry_size]), enqueued on `stream`"""
        _check(lib().b200dpf_update_rows_device(self.handle, C.c_void_p(idx_ptr), C.c_void_p(rows_ptr), count,
                                                C.c_void_p(stream)), "b200dpf_update_rows_device")

    def set_option(self, name, value):
        _check(lib().b200dpf_ctx_set_option(self.handle, name.encode(), int(value)), "b200dpf_ctx_set_option")

    def read_timing(self, max_blocks=1024):
        """[blocks, 8] uint64 %globaltimer stamps of the last evaluation (option "timing" = 1)"""
        buf = np.zeros((max_blocks, 8), np.uint64)
        n = C.c_int()
        _check(lib().b200dpf_ctx_read_timing(self.handle, buf, max_blocks, C.byref(n)), "b200dpf_ctx_read_timing")
        return buf[:n.value]

    def eval_device(self, keys_ptr, nkeys, prf, out_ptr, stream=0, accumulate=False):
        fn = lib().b200dpf_eval_device_acc if accumulate else lib().b200dpf_eval_device
        _check(fn(self.handle, C.c_void_p(keys_ptr), nkeys, prf, C.c_void_p(out_ptr),
                                         C.c_void_p(stream)), "b200dpf_eval_device")

    def expand_device(self, keys_ptr, nkeys, prf, out_ptr, stream=0):
        _check(lib().b200dpf_expand_device(self.handle, C.c_void_p(keys_ptr), nkeys, prf, C.c_void_p(out_ptr),
                                           C.c_void_p(stream)), "b200dpf_expand_device")

    def set_subtree_log2(self, s):
        _check(lib().b200dpf_ctx_set_subtree_log2(self.handle, s), "b200dpf_ctx_set_subtree_log2")

    @property
    def last_device_ms(self):
        return lib().b200dpf_ctx_last_device_ms(self.handle)

    @property
    def last_launches(self):
        return lib().b200dpf_ctx_last_launches(self.handle)

    @property
    def rows_per_leaf(self):
        return lib().b200dpf_ctx_rows_per_leaf(self.handle)

    @property
    def trimmed(self):
        return lib().b200dpf_ctx_trimmed(self.handle) == 1

    @property
    def table_rows(self):
        """rows of the device table, padding included (b200dpf_ctx_table_rows)"""
        return lib().b200dpf_ctx_table_rows(self.handle)

    def close(self):
        if self.handle:
            lib().b200dpf_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GroupContext(Context):
    """Many tables ("bins") of one entry size behind one context: the batch-PIR front end
    (b200dpf_group_create / b200dpf_group_eval).  early_termination=True makes the context for
    early-terminated keys (b200dpf_group_create_et): bins of >= 8 rows, four rows per tree leaf.  xor=True
    makes it for XOR-shared keys (b200dpf_group_create_xor): bins of >= 256 rows, 128 rows per tree leaf,
    and results that XOR (not add) to the selected row.  trimmed=True makes a trimmed grouped context
    (b200dpf_group_create_trimmed) of the kind: bins of any size, numbered as on a trimmed Context."""

    def __init__(self, tables, device=0, early_termination=False, xor=False, trimmed=False):
        if xor and early_termination:
            raise ValueError("a context takes one kind of key: pass xor=True or early_termination=True, not both")
        self.tables = [np.ascontiguousarray(t, np.int32) for t in tables]
        assert all(t.ndim == 2 and t.shape[1] == self.tables[0].shape[1] for t in self.tables)
        self.entry_size = self.tables[0].shape[1]
        self.n = max(t.shape[0] for t in self.tables)
        sizes = np.array([t.shape[0] for t in self.tables], np.int64)
        ptrs = (C.c_void_p * len(self.tables))(*[t.ctypes.data for t in self.tables])
        self.handle = C.c_void_p()
        self.kind = "_xor" if xor else "_et" if early_termination else ""
        self._trimmed = trimmed        # what pack_queries needs besides the kind and the bin sizes
        if trimmed:
            _check(lib().b200dpf_group_create_trimmed(C.byref(self.handle), ptrs, sizes, len(self.tables), self.entry_size,
                                                      device, KIND_IDS[self.kind]), "b200dpf_group_create_trimmed")
            return
        name = "b200dpf_group_create" + self.kind
        _check(getattr(lib(), name)(C.byref(self.handle), ptrs, sizes, len(self.tables), self.entry_size, device), name)

    @property
    def nbins(self):
        return lib().b200dpf_group_bins(self.handle)

    @property
    def bin_rows(self):
        """the live rows of each bin"""
        return [t.shape[0] for t in self.tables]

    def eval(self, keys, bins, prf):
        keys = np.ascontiguousarray(keys, np.int32).reshape(-1, KEY_WORDS)
        bins = np.ascontiguousarray(bins, np.int32)
        assert bins.shape == (keys.shape[0],)
        out = np.zeros((keys.shape[0], self.entry_size), np.int32)
        _check(lib().b200dpf_group_eval(self.handle, keys, bins, keys.shape[0], prf, out), "b200dpf_group_eval")
        return out

    def eval_device(self, keys_ptr, bins, prf, out_ptr, stream=0):
        """eval from device keys (int32 [len(bins), 524] at keys_ptr) into device results (int32
        [len(bins), entry_size] at out_ptr), enqueued on `stream` with no host synchronisation.  `bins` stays
        on the host: the launch is planned from it."""
        bins = np.ascontiguousarray(bins, np.int32).reshape(-1)
        _check(lib().b200dpf_group_eval_device(self.handle, C.c_void_p(keys_ptr), bins, len(bins), prf,
                                               C.c_void_p(out_ptr), C.c_void_p(stream)), "b200dpf_group_eval_device")

    def eval_device_bins(self, keys_ptr, bins_ptr, nkeys, prf, out_ptr, bad_ptr=0, stream=0):
        """eval_device with the bins in device memory too (int32 [nkeys] at bins_ptr), planned on the GPU and
        enqueued on `stream` without any host wait.  A key whose bin is outside [0, nbins) gets a zero row; if
        bad_ptr is not 0, the int64 there receives the number of such keys."""
        _check(lib().b200dpf_group_eval_device_bins(self.handle, C.c_void_p(keys_ptr), C.c_void_p(bins_ptr), nkeys, prf,
                                                    C.c_void_p(out_ptr), C.c_void_p(bad_ptr or None), C.c_void_p(stream)),
               "b200dpf_group_eval_device_bins")

    def plan_lists(self, device_planned):
        """for tests: the lists of the last plan, made on the device by eval_device_bins (device_planned=True) or on the
        host by eval / eval_device: (counts, descs, units, order) with counts = (key groups, work units, keys, keys
        whose bin is out of range), descs uint32 [K, 8], units uint32 [U, 4], order uint32 [nkeys, 2]"""
        counts = np.zeros(4, np.int64)
        empty = np.zeros(8, np.uint32)
        which = 0 if device_planned else 1
        _check(lib().b200dpf_group_plan_lists(self.handle, which, counts, empty.ctypes.data, 0, empty.ctypes.data, 0,
                                              empty.ctypes.data, 0), "b200dpf_group_plan_lists")
        descs = np.zeros((max(int(counts[0]), 1), 8), np.uint32)
        units = np.zeros((max(int(counts[1]), 1), 4), np.uint32)
        order = np.zeros((max(int(counts[2]), 1), 2), np.uint32)
        _check(lib().b200dpf_group_plan_lists(self.handle, which, counts, descs.ctypes.data, int(counts[0]), units.ctypes.data,
                                              int(counts[1]), order.ctypes.data, int(counts[2])), "b200dpf_group_plan_lists")
        return counts, descs[:counts[0]], units[:counts[1]], order[:counts[2]]

    @property
    def query_bytes(self):
        """bytes of one compact query (pack_queries): one compact key per bin, at the bin's depth"""
        return lib().b200dpf_group_query_bytes(self.handle)

    def eval_queries_device(self, keys_ptr, nqueries, prf, out_ptr, stream=0, compact=False):
        """batch-PIR queries of one key per bin from device memory into device results (int32 [nqueries, nbins,
        entry_size] at out_ptr), enqueued on `stream` with no host synchronisation.  keys_ptr holds int32
        [nqueries, nbins, 524] wire-format keys, or with compact=True uint8 [nqueries, query_bytes] compact
        queries (pack_queries).  The launch plan depends on nqueries alone and is reused while nqueries, prf
        and the options stay those of the previous call."""
        fmt = KEYS_COMPACT if compact else KEYS_WIRE
        _check(lib().b200dpf_group_eval_queries_device(self.handle, C.c_void_p(keys_ptr), fmt, nqueries, prf,
                                                       C.c_void_p(out_ptr), C.c_void_p(stream)),
               "b200dpf_group_eval_queries_device")

    def gen_queries_device(self, alphas_ptr, seeds_ptr, nqueries, prf, out_a_ptr, out_b_ptr, stream=0, compact=False):
        """both servers' batch-PIR queries for eval_queries_device, made on the GPU from device buffers and
        enqueued on `stream` with no host synchronisation: alphas_ptr int64 [nqueries, nbins] (the row of bin g
        query q selects, taken mod the bin's size), seeds_ptr uint8 [nqueries, nbins, 44] (entropy from a
        CSPRNG).  out_a_ptr / out_b_ptr receive int32 [nqueries, nbins, 524] wire-format keys, or with
        compact=True uint8 [nqueries, query_bytes] compact queries; key (q, g) is gen_batch<kind>'s for the same
        row, bin size and seed (and pack_queries' bytes of it)."""
        fmt = KEYS_COMPACT if compact else KEYS_WIRE
        _check(lib().b200dpf_group_gen_queries_device(self.handle, C.c_void_p(alphas_ptr), C.c_void_p(seeds_ptr), nqueries,
                                                      prf, fmt, C.c_void_p(out_a_ptr), C.c_void_p(out_b_ptr),
                                                      C.c_void_p(stream)),
               "b200dpf_group_gen_queries_device")

    def pack_queries(self, keys):
        """int32 [Q, nbins, 524] wire-format keys (key g of query q for bin g) -> uint8 [Q, query_bytes] compact
        queries: each query its keys' compact forms (key_pack of the context's kind) back to back.  A key that
        is not of the context's kind, or not for its bin's size, raises."""
        keys = np.ascontiguousarray(keys, np.int32)
        nbins = len(self.bin_rows)
        if keys.ndim != 3 or keys.shape[1:] != (nbins, KEY_WORDS):
            raise ValueError("pack_queries: keys must be int32 [Q, %d, %d], got shape %s" % (nbins, KEY_WORDS, keys.shape))
        lane_bits = KINDS[self.kind][0]
        trimmed = getattr(self, "_trimmed", False)
        domains = [trimmed_domain(rows, self.kind) if trimmed else rows for rows in self.bin_rows]
        sizes = [lib().b200dpf_key_packed_size(n.bit_length() - 1 - lane_bits) for n in domains]
        out = np.empty((keys.shape[0], sum(sizes)), np.uint8)
        for q in range(keys.shape[0]):
            off = 0
            for g, size in enumerate(sizes):
                packed = _key_pack(self.kind, keys[q, g])
                if len(packed) != size:
                    raise ValueError("pack_queries: key %d of query %d is for another bin size (%d packed bytes, bin %d "
                                     "takes %d)" % (g, q, len(packed), g, size))
                out[q, off:off + size] = np.frombuffer(packed, np.uint8)
                off += size
        return out

    def update_rows(self, bins, indices, rows):
        """row indices[j] of bin bins[j] := rows[j] (last occurrence wins); synchronous"""
        bins = np.ascontiguousarray(bins, np.int32).reshape(-1)
        indices = np.ascontiguousarray(indices, np.int64).reshape(-1)
        assert bins.shape == indices.shape
        rows = np.ascontiguousarray(rows, np.int32).reshape(len(indices), self.entry_size)
        _check(lib().b200dpf_group_update_rows(self.handle, bins, indices, rows, len(indices)), "b200dpf_group_update_rows")


def _layout_args(n, nbins, seed):
    return int(n), int(nbins), int(seed) & 0xFFFFFFFFFFFFFFFF


def batchcode_locate(n, nbins, seed, row):
    """(bins, rows): the bin and the in-bin row of copies 0, 1, 2 of `row` in the batch-code layout (n, nbins, seed)
    (b200dpf_batchcode_locate); host only"""
    bins = np.zeros(3, np.int32)
    rows = np.zeros(3, np.int64)
    _check(lib().b200dpf_batchcode_locate(*_layout_args(n, nbins, seed), int(row), bins, rows), "b200dpf_batchcode_locate")
    return bins, rows


def batchcode_plan(n, nbins, seed, wanted):
    """the client's plan of queries of k wanted rows (b200dpf_batchcode_plan): wanted int64 [Q, k] -> (alphas int64
    [Q, nbins], the in-bin row to query in each bin; slots int32 [Q, k], the bin answering wanted row i or -1)"""
    wanted = np.ascontiguousarray(wanted, np.int64)
    if wanted.ndim != 2:
        raise ValueError("batchcode_plan: wanted must be [Q, k], got shape %s" % (wanted.shape,))
    alphas = np.zeros((wanted.shape[0], max(int(nbins), 0)), np.int64)
    slots = np.zeros(wanted.shape, np.int32)
    _check(lib().b200dpf_batchcode_plan(*_layout_args(n, nbins, seed), wanted, wanted.shape[0], wanted.shape[1], alphas, slots),
           "b200dpf_batchcode_plan")
    return alphas, slots


class BatchCodeContext(GroupContext):
    """One table of n rows stored as a batch code (b200dpf_batchcode_create): every row in 3 of nbins trimmed bins, so a
    query of one key per bin retrieves any k rows the client's plan (batchcode_plan) places.  The kinds as for
    GroupContext; every GroupContext evaluation works on it.  Rows change through update_rows, all three copies at once."""

    def __init__(self, table, nbins, seed, device=0, early_termination=False, xor=False):
        if xor and early_termination:
            raise ValueError("a context takes one kind of key: pass xor=True or early_termination=True, not both")
        table = np.ascontiguousarray(table, np.int32)
        if table.ndim != 2:
            raise ValueError("BatchCodeContext: table must be [n, entry_size], got shape %s" % (table.shape,))
        self.n, self.entry_size = table.shape
        self.kind = "_xor" if xor else "_et" if early_termination else ""
        self._trimmed = True
        self.handle = C.c_void_p()
        _check(lib().b200dpf_batchcode_create(C.byref(self.handle), table.ctypes.data_as(C.c_void_p), self.n, self.entry_size,
                                              int(nbins), int(seed) & 0xFFFFFFFFFFFFFFFF, device, KIND_IDS[self.kind]),
               "b200dpf_batchcode_create")

    @property
    def layout(self):
        """(n, nbins, seed): the public parameters a client plans with (b200dpf_batchcode_layout)"""
        n, nbins, seed = C.c_int64(), C.c_int(), C.c_uint64()
        _check(lib().b200dpf_batchcode_layout(self.handle, C.byref(n), C.byref(nbins), C.byref(seed)), "b200dpf_batchcode_layout")
        return n.value, nbins.value, seed.value

    @property
    def bin_rows(self):
        """the rows of each bin: 3 m_j, m_j = ceil((n - j) / nbins)"""
        n, nbins, _ = self.layout
        return [3 * ((n - j + nbins - 1) // nbins) for j in range(nbins)]

    def plan_device(self, wanted_ptr, nqueries, k, alphas_ptr, slots_ptr, stream=0):
        """batchcode_plan on the GPU from device buffers (wanted int64 [nqueries, k] into alphas int64 [nqueries,
        nbins] and slots int32 [nqueries, k]), enqueued on `stream` with no host wait"""
        _check(lib().b200dpf_batchcode_plan_device(self.handle, C.c_void_p(wanted_ptr), nqueries, k, C.c_void_p(alphas_ptr),
                                                   C.c_void_p(slots_ptr), C.c_void_p(stream)), "b200dpf_batchcode_plan_device")

    def update_rows(self, indices, rows):
        """table[indices[j]] := rows[j] in all three copies (last occurrence wins); synchronous"""
        indices = np.ascontiguousarray(indices, np.int64).reshape(-1)
        rows = np.ascontiguousarray(rows, np.int32).reshape(len(indices), self.entry_size)
        _check(lib().b200dpf_batchcode_update_rows(self.handle, indices, rows, len(indices)), "b200dpf_batchcode_update_rows")


def kwpir_locate(m, seed, keywords):
    """the in-bin rows int64 [Q, 3] to query for keywords [Q] in the keyword-PIR layout (m, seed): row c of keyword j is
    h_c(keywords[j]) (b200dpf_kwpir_locate); host only"""
    keywords = np.ascontiguousarray(keywords, np.uint64).reshape(-1)
    rows = np.zeros((len(keywords), 3), np.int64)
    _check(lib().b200dpf_kwpir_locate(int(m), int(seed) & 0xFFFFFFFFFFFFFFFF, keywords, len(keywords), rows), "b200dpf_kwpir_locate")
    return rows


class KeywordContext(GroupContext):
    """(keyword, value) items in a cuckoo hash table of three trimmed bins of m slots (b200dpf_kwpir_create): a query of
    one key per bin, for the keyword's rows kwpir_locate gives, returns the value with its tag.  keywords: uint64 [n],
    values: int32 [n, value_size]; bins of value_size + 2 columns.  The kinds as for GroupContext; every GroupContext
    evaluation works on it.  Values change through update.  Raises B200DPFError "... failed (-5)" (EFULL) when the
    placement does not finish with this seed (dpf.KeywordDPF retries further seeds)."""

    def __init__(self, keywords, values, m, seed, device=0, early_termination=False, xor=False):
        if xor and early_termination:
            raise ValueError("a context takes one kind of key: pass xor=True or early_termination=True, not both")
        keywords = np.ascontiguousarray(keywords, np.uint64).reshape(-1)
        values = np.ascontiguousarray(values, np.int32)
        if values.ndim != 2 or values.shape[0] != len(keywords):
            raise ValueError("KeywordContext: values must be [n, value_size] with one row per keyword, got shape %s" % (values.shape,))
        self.n, self.value_size = values.shape
        self.entry_size = self.value_size + 2
        self.kind = "_xor" if xor else "_et" if early_termination else ""
        self._trimmed = True
        self.handle = C.c_void_p()
        _check(lib().b200dpf_kwpir_create(C.byref(self.handle), keywords.ctypes.data_as(C.c_void_p), values.ctypes.data_as(C.c_void_p),
                                          self.n, self.value_size, int(m), int(seed) & 0xFFFFFFFFFFFFFFFF, device, KIND_IDS[self.kind]),
               "b200dpf_kwpir_create")

    @property
    def layout(self):
        """(n, m, seed, value_size): the public parameters a client locates with (b200dpf_kwpir_layout)"""
        n, m, seed, e = C.c_int64(), C.c_int64(), C.c_uint64(), C.c_int()
        _check(lib().b200dpf_kwpir_layout(self.handle, C.byref(n), C.byref(m), C.byref(seed), C.byref(e)), "b200dpf_kwpir_layout")
        return n.value, m.value, seed.value, e.value

    @property
    def build_stats(self):
        """(rounds, ms): the rounds the placement took and their device time (b200dpf_kwpir_build_stats)"""
        rounds, ms = C.c_int(), C.c_double()
        _check(lib().b200dpf_kwpir_build_stats(self.handle, C.byref(rounds), C.byref(ms)), "b200dpf_kwpir_build_stats")
        return rounds.value, ms.value

    @property
    def bin_rows(self):
        """the rows of each bin: m"""
        return [self.layout[1]] * 3

    def tags(self):
        """uint64 [3, m]: the tag stored in every slot, keyword + 1 or 0 for an empty slot (b200dpf_kwpir_tags)"""
        out = np.zeros((3, self.layout[1]), np.uint64)
        _check(lib().b200dpf_kwpir_tags(self.handle, out), "b200dpf_kwpir_tags")
        return out

    def plan_device(self, keywords_ptr, nqueries, alphas_ptr, stream=0):
        """kwpir_locate on the GPU from device buffers (keywords uint64 [nqueries] into alphas int64 [nqueries, 3]),
        enqueued on `stream` with no host wait"""
        _check(lib().b200dpf_kwpir_plan_device(self.handle, C.c_void_p(keywords_ptr), nqueries, C.c_void_p(alphas_ptr),
                                               C.c_void_p(stream)), "b200dpf_kwpir_plan_device")

    def update(self, keywords, values):
        """the value of keywords[j] := values[j] (last occurrence wins); synchronous.  A keyword not in the table raises,
        and nothing is applied."""
        keywords = np.ascontiguousarray(keywords, np.uint64).reshape(-1)
        values = np.ascontiguousarray(values, np.int32).reshape(len(keywords), self.value_size)
        _check(lib().b200dpf_kwpir_update(self.handle, keywords, values, len(keywords)), "b200dpf_kwpir_update")
