"""ctypes doorway onto the CPU oracle -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs may import this module.  The product package
(gpu-dpf_b200/) must never do so.

Two libraries live behind it:

* ``Oracle``  -> oracle/libdpforacle.so, our plain-C restatement (dpf_oracle.c);
* ``Ref``     -> oracle/_ref/libdpfref.so, the unmodified reference CPU core
  (dpf_base/dpf.h) behind oracle/ref_shim.cc.  Present wherever ``make -C
  oracle ref`` ran with the reference tree available (the build container),
  and shipped prebuilt to the GPU box with the gpurun snapshot.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_WORDS = 524
PRF_DUMMY, PRF_SALSA20, PRF_CHACHA20, PRF_AES128 = 0, 1, 2, 3
PRF_NAMES = {0: "DUMMY", 1: "SALSA20", 2: "CHACHA20", 3: "AES128"}

_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(dtype=np.int64, flags="C_CONTIGUOUS")


def build(ref=True):
    """(Re)build the oracle, and oracle/_ref when the reference tree is here."""
    subprocess.run(["make", "-s", "-C", HERE, "oracle"], check=True)
    if ref:
        subprocess.run(["make", "-s", "-C", HERE, "ref"], check=True)


def _u128(lo, hi):
    return (int(hi) << 64) | int(lo)


class Oracle:
    """Our C restatement."""

    # the newest entry points: a library without them was built from older sources
    REQUIRED = ("orc_eval_points", "orc_eval_points_et")

    def __init__(self):
        path = os.path.join(HERE, "libdpforacle.so")
        if not os.path.exists(path):
            build(ref=False)
        L = self.lib = C.CDLL(path)
        missing = [s for s in self.REQUIRED if not hasattr(L, s)]
        if missing:
            raise RuntimeError("%s is stale (no %s): rebuild it with `make -C %s oracle`"
                               % (path, ", ".join(missing), HERE))
        u64p = C.POINTER(C.c_uint64)
        L.orc_prf.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint32, u64p, u64p]
        L.orc_aes128_encrypt.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p]
        L.orc_eval_flat.argtypes = [_i32p, C.c_int64, C.c_int, u64p, u64p]
        L.orc_eval_full_flat.argtypes = [_i32p, C.c_int, _i32p]
        L.orc_eval_full_tree.argtypes = [_i32p, C.c_int, _i32p]
        L.orc_eval_dot.argtypes = [_i32p, C.c_int64, C.c_int, _i32p, C.c_int64, C.c_int, C.c_int, _i32p]
        L.orc_eval_dot_range.argtypes = [_i32p, C.c_int64, C.c_int, _i32p, C.c_int64, C.c_int,
                                         C.c_int64, C.c_int64, _i32p]
        L.orc_eval_dot_shard.argtypes = [_i32p, C.c_int, _i32p, C.c_int64, C.c_int, C.c_int64, C.c_int64, _i32p]
        L.orc_gen.argtypes = [C.c_int64, C.c_int64, C.c_uint32, C.c_int, _i32p, _i32p]
        L.orc_bitrev.argtypes = [C.c_uint32, C.c_int]
        L.orc_bitrev.restype = C.c_uint32
        for name in self.REQUIRED:
            getattr(L, name).argtypes = [_i32p, C.c_int64, C.c_int, _i64p, C.c_int64, C.c_int, _i32p]

    def _points(self, fn, keys, prf, points, width, nthreads):
        keys = np.ascontiguousarray(keys, np.int32).reshape(-1, KEY_WORDS)
        points = np.ascontiguousarray(points, np.int64).reshape(-1)
        out = np.zeros((keys.shape[0], points.size * width), np.int32)
        rc = fn(keys, keys.shape[0], prf, points, points.size, nthreads or os.cpu_count() or 1, out)
        assert rc == 0, rc
        return out

    def eval_points(self, keys, prf, idx, nthreads=0):
        """int32 [B, len(idx)]: low 32 bits of EvaluateFlat(keys[b], idx[j]), one walk per value,
        on `nthreads` host threads (0 = every core)"""
        return self._points(self.lib.orc_eval_points, keys, prf, idx, 1, nthreads)

    def eval_points_et(self, keys, prf, leaves, nthreads=0):
        """early-terminated keys: int32 [B, 4 * len(leaves)], the four words of each leaf in turn
        (the shares of rows 4 * leaf .. 4 * leaf + 3)"""
        return self._points(self.lib.orc_eval_points_et, keys, prf, leaves, 4, nthreads)

    def prf(self, prf, seed, pos):
        lo, hi = C.c_uint64(), C.c_uint64()
        self.lib.orc_prf(prf, seed & (2**64 - 1), seed >> 64, pos, C.byref(lo), C.byref(hi))
        return _u128(lo.value, hi.value)

    def aes128_encrypt(self, key, block):
        out = C.create_string_buffer(16)
        self.lib.orc_aes128_encrypt(bytes(key), bytes(block), out)
        return out.raw

    def gen(self, alpha, n, seed32, prf):
        a = np.zeros(KEY_WORDS, np.int32)
        b = np.zeros(KEY_WORDS, np.int32)
        rc = self.lib.orc_gen(alpha, n, seed32 & 0xFFFFFFFF, prf, a, b)
        if rc:
            raise ValueError("orc_gen rc=%d" % rc)
        return a, b

    def eval_flat(self, key, idx, prf):
        lo, hi = C.c_uint64(), C.c_uint64()
        self.lib.orc_eval_flat(np.ascontiguousarray(key, np.int32), idx, prf, C.byref(lo), C.byref(hi))
        return _u128(lo.value, hi.value)

    def eval_full(self, key, prf, tree=True):
        key = np.ascontiguousarray(key, np.int32)
        n = int(key[130 * 4])
        out = np.zeros(n, np.int32)
        fn = self.lib.orc_eval_full_tree if tree else self.lib.orc_eval_full_flat
        rc = fn(key, prf, out)
        assert rc == 0
        return out

    def eval_dot(self, keys, prf, table, tree=True):
        keys = np.ascontiguousarray(keys, np.int32).reshape(-1, KEY_WORDS)
        table = np.ascontiguousarray(table, np.int32)
        n, e = table.shape
        out = np.zeros((keys.shape[0], e), np.int32)
        rc = self.lib.orc_eval_dot(keys, keys.shape[0], prf, table, n, e, 1 if tree else 0, out)
        assert rc == 0, rc
        return out

    def eval_dot_range(self, keys, prf, table, idx_begin, idx_count):
        keys = np.ascontiguousarray(keys, np.int32).reshape(-1, KEY_WORDS)
        table = np.ascontiguousarray(table, np.int32)
        n, e = table.shape
        out = np.zeros((keys.shape[0], e), np.int32)
        rc = self.lib.orc_eval_dot_range(keys, keys.shape[0], prf, table, n, e, idx_begin, idx_count, out)
        assert rc == 0, rc
        return out

    def eval_dot_shard(self, key, prf, table, pos_begin, pos_count):
        key = np.ascontiguousarray(key, np.int32)
        table = np.ascontiguousarray(table, np.int32)
        n, e = table.shape
        out = np.zeros(e, np.int32)
        rc = self.lib.orc_eval_dot_shard(key, prf, table, n, e, pos_begin, pos_count, out)
        assert rc == 0, rc
        return out

    def bitrev(self, x, bits):
        return int(self.lib.orc_bitrev(x, bits))


class Ref:
    """The unmodified reference CPU core (oracle/_ref/libdpfref.so)."""

    PATH = os.path.join(HERE, "_ref", "libdpfref.so")

    @classmethod
    def available(cls):
        return os.path.exists(cls.PATH)

    def __init__(self):
        if not self.available():
            raise FileNotFoundError(self.PATH)
        L = self.lib = C.CDLL(self.PATH)
        u64p = C.POINTER(C.c_uint64)
        L.ref_prf.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint32, u64p, u64p]
        L.ref_gen.argtypes = [C.c_int64, C.c_int64, C.c_uint32, C.c_int, _i32p, _i32p]
        L.ref_eval_flat.argtypes = [_i32p, C.c_int64, C.c_int, u64p, u64p]
        L.ref_eval_full.argtypes = [_i32p, C.c_int, _i32p]
        L.ref_eval_dot_mt.argtypes = [_i32p, C.c_int64, C.c_int, _i32p, C.c_int64, C.c_int,
                                      C.c_int64, C.c_int64, C.c_int, _i32p]

    def prf(self, prf, seed, pos):
        lo, hi = C.c_uint64(), C.c_uint64()
        self.lib.ref_prf(prf, seed & (2**64 - 1), seed >> 64, pos, C.byref(lo), C.byref(hi))
        return _u128(lo.value, hi.value)

    def gen(self, alpha, n, seed32, prf):
        a = np.zeros(KEY_WORDS, np.int32)
        b = np.zeros(KEY_WORDS, np.int32)
        self.lib.ref_gen(alpha, n, seed32 & 0xFFFFFFFF, prf, a, b)
        return a, b

    def eval_flat(self, key, idx, prf):
        lo, hi = C.c_uint64(), C.c_uint64()
        self.lib.ref_eval_flat(np.ascontiguousarray(key, np.int32), idx, prf, C.byref(lo), C.byref(hi))
        return _u128(lo.value, hi.value)

    def eval_full(self, key, prf):
        key = np.ascontiguousarray(key, np.int32)
        n = int(key[130 * 4])
        out = np.zeros(n, np.int32)
        self.lib.ref_eval_full(key, prf, out)
        return out

    def eval_dot_mt(self, keys, prf, table, idx_begin, idx_count, nthreads):
        keys = np.ascontiguousarray(keys, np.int32).reshape(-1, KEY_WORDS)
        table = np.ascontiguousarray(table, np.int32)
        n, e = table.shape
        out = np.zeros((keys.shape[0], e), np.int32)
        self.lib.ref_eval_dot_mt(keys, keys.shape[0], prf, table, n, e, idx_begin, idx_count, nthreads, out)
        return out
