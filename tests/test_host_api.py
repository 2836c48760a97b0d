"""CPU-side product code (keygen, eval_cpu, the C-ABI surface, the dpf.DPF API)
against the oracle and the golden vectors.  No GPU; no compute calls on the GPU
entry points beyond checking that they refuse to run without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import b200dpf
from common import formula_table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "b200dpf.h")).read()
    declared = sorted(set(re.findall(r"\b(b200dpf_[a-z0-9_]+)\s*\(", header)) - {"b200dpf_ctx"})
    assert declared == sorted(b200dpf.SYMBOLS)
    L = C.CDLL(b200dpf.LIB_PATH)
    for name in declared:
        assert hasattr(L, name), name
    assert b"sm_90a" in b200dpf.lib().b200dpf_version()


def test_gen_matches_golden_keys(golden):
    for ci, (prf, n, alpha, seed32) in enumerate(golden["case_meta"]):
        ka, kb = b200dpf.gen(int(alpha), int(n), int(seed32), int(prf))
        assert np.array_equal(ka, golden["keys_a"][ci])
        assert np.array_equal(kb, golden["keys_b"][ci])


def test_gen_batch_matches_gen(oracle):
    n, prf = 4096, 3
    alphas = [0, 1, 17, 4095, 2048, 999]
    seeds = [5, 6, 7, 8, 9, 2**32 - 1]
    a, b = b200dpf.gen_batch(alphas, n, seeds, prf, nthreads=3)
    for i in range(len(alphas)):
        oa, ob = oracle.gen(alphas[i], n, seeds[i], prf)
        assert np.array_equal(a[i], oa) and np.array_equal(b[i], ob)


def test_gen_secure(oracle):
    """ChaCha20-DRBG keygen: valid keys (shares reconstruct the point function, the oracle agrees
    on the share vector), deterministic in the seed, sensitive to all of it, full-width words."""
    seed = bytes(range(44))
    for prf in range(4):
        for n, alpha in ((2, 1), (1024, 77), (1 << 15, 31337)):
            ka, kb = b200dpf.gen_secure(alpha, n, seed, prf)
            sa, sb = b200dpf.eval_cpu(ka, prf), b200dpf.eval_cpu(kb, prf)
            d = (sa.astype(np.int64) - sb.astype(np.int64)) % (1 << 32)
            assert d[alpha] == 1 and np.count_nonzero(d) == 1
            assert np.array_equal(sa, oracle.eval_full(ka, prf))
    k1, _ = b200dpf.gen_secure(5, 1024, seed, 3)
    k2, _ = b200dpf.gen_secure(5, 1024, seed, 3)
    k3, _ = b200dpf.gen_secure(5, 1024, seed[:43] + b"\xff", 3)
    assert np.array_equal(k1, k2) and not np.array_equal(k1, k3)
    # upper-level correction words are 128-bit here (32-bit in the reference generator)
    cw_top = k1[4:8]
    assert np.any(cw_top[1:] != 0)
    with pytest.raises(b200dpf.B200DPFError, match="44 bytes"):
        b200dpf.gen_secure(5, 1024, b"short", 3)
    # the exact keys (the DRBG against RFC 8439's vectors, the construction against the reference's keys) are
    # checked in tests/test_keygen_ref_host.py


def test_eval_cpu_matches_golden_and_oracle(oracle, golden):
    for ci, (prf, n, alpha, seed32) in enumerate(golden["case_meta"]):
        prf, n = int(prf), int(n)
        got = b200dpf.eval_cpu(golden["keys_a"][ci], prf)
        if n <= 1024:
            assert np.array_equal(got, golden["share_a_%d" % ci])
        assert np.array_equal(got, oracle.eval_full(golden["keys_a"][ci], prf))


def test_eval_cpu_large_domain(oracle):
    """n = 2^18: walks across several 2^16-leaf subtrees of the shared traversal code."""
    n = 1 << 18
    for prf in (0, 2):
        ka, kb = b200dpf.gen(123457, n, 77, prf)
        sa, sb = b200dpf.eval_cpu(ka, prf), b200dpf.eval_cpu(kb, prf)
        d = (sa.astype(np.int64) - sb.astype(np.int64)) % (1 << 32)
        assert d[123457] == 1 and np.count_nonzero(d) == 1
        assert np.array_equal(sa, oracle.eval_full(ka, prf))


def test_error_codes():
    L = b200dpf.lib()
    a = np.zeros(524, np.int32)
    b = np.zeros(524, np.int32)
    assert L.b200dpf_gen(5, 100, b"abcd", 4, 3, a, b) == -1          # n not a power of two
    assert L.b200dpf_gen(128, 128, b"abcd", 4, 3, a, b) == -1        # alpha >= n
    assert L.b200dpf_gen(1, 128, b"abcd", 4, 9, a, b) == -1          # bad prf
    assert b"power-of-two" in L.b200dpf_last_error()
    assert L.b200dpf_eval_cpu(a, 3, np.zeros(4, np.int32)) == -1     # all-zero key is malformed
    assert L.b200dpf_key_n(a) == -1


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-device behaviour")
def test_gpu_entry_points_fail_loudly_without_device():
    with pytest.raises(b200dpf.B200DPFError, match="no CUDA device"):
        b200dpf.Context(formula_table(128, 16))


def test_python_api_cpu_side():
    import dpf
    import dpf_cpp
    assert (dpf_cpp.ENTRY_SIZE, dpf_cpp.BATCH_SIZE) == (16, 512)
    assert (dpf_cpp.PRF_DUMMY, dpf_cpp.PRF_SALSA20, dpf_cpp.PRF_CHACHA20, dpf_cpp.PRF_AES128) == (0, 1, 2, 3)
    for name in ("gen", "eval_cpu", "eval_gpu", "eval_init", "eval_free"):
        assert callable(getattr(dpf_cpp, name))
    d = dpf.DPF()
    assert repr(d) == "DPF(_uninitialized_, prf_method=AES128)"
    with pytest.raises(Exception, match="power of two"):
        d.gen(3, 100)
    with pytest.raises(Exception, match="must be less than n"):
        d.gen(128, 128)
    with pytest.raises(Exception, match="Must call `eval_init`"):
        d.eval_gpu([])
    with pytest.raises(Exception, match="at least 128"):
        d.eval_init(torch.zeros(64, 16).int())
    with pytest.raises(Exception, match="power of two"):
        d.eval_init(torch.zeros(192, 16).int())
    k1, k2 = d.gen(42, 1024)
    assert k1.dtype == torch.int32 and tuple(k1.shape) == (524,)
    v = d.eval_cpu([k1], one_hot_only=True) - d.eval_cpu([k2], one_hot_only=True)
    assert v[0, 42] == 1 and v.count_nonzero() == 1
    dpf.test_cpu_dpf_one_hot()
    dpf.test_cpu_dpf()


def test_secure_keygen_is_the_default(oracle):
    """dpf.DPF.gen / gen_batch without a seed use the ChaCha20 DRBG (full-width correction words); an explicit seed
    keeps the reference's 32-bit generator so golden/parity keys stay bit-identical."""
    import os
    import dpf
    d = dpf.DPF(prf=dpf.DPF.PRF_CHACHA20)
    n = 4096
    k1, k2 = d.gen(77, n)
    # the reference draws the upper-level cw_1 words as 32-bit values (dpf.h:450): such slots have words 1..3 zero

    def narrow_slots(key):
        cw1 = key.numpy().reshape(131, 4)[1:1 + 2 * 12]
        return int(((cw1[:, 0] != 0) & (cw1[:, 1:] == 0).all(axis=1)).sum())
    assert narrow_slots(k1) == 0
    v = oracle.eval_full(k1.numpy(), 2).astype(np.uint32) - oracle.eval_full(k2.numpy(), 2).astype(np.uint32)
    assert v[77] == 1 and np.count_nonzero(v) == 1
    legacy1, _ = d.gen(77, n, seed=b"\x01\x02\x03\x04" + bytes(124))
    legacy2, _ = d.gen(77, n, seed=b"\x01\x02\x03\x04" + bytes(124))
    want, _ = b200dpf.gen(77, n, 0x04030201, 2)
    assert torch.equal(legacy1, legacy2) and np.array_equal(legacy1.numpy(), want)
    assert narrow_slots(legacy1) > 0
    ka, kb = d.gen_batch([1, 2, 4095], n)
    for i, idx in enumerate([1, 2, 4095]):
        v = oracle.eval_full(ka[i].numpy(), 2).astype(np.uint32) - oracle.eval_full(kb[i].numpy(), 2).astype(np.uint32)
        assert v[idx] == 1 and np.count_nonzero(v) == 1
    assert not torch.equal(ka, d.gen_batch([1, 2, 4095], n)[0])          # fresh entropy every call
    sa, _ = b200dpf.gen_batch_secure([9, 10], n, bytes(range(88)), 2)
    one, _ = b200dpf.gen_secure(10, n, bytes(range(44, 88)), 2)
    assert np.array_equal(sa[1], one)


def test_compact_key_format(golden):
    """pack/unpack round-trips every golden key exactly and shrinks it to 32 + 64*depth bytes, every field
    16-byte aligned (the GPU reads this form in place: b200dpf_eval_packed)."""
    import dpf_cpp
    for ci, (prf, n, alpha, seed32) in enumerate(golden["case_meta"]):
        for keys in (golden["keys_a"], golden["keys_b"]):
            k = keys[ci]
            packed = b200dpf.key_pack(k)
            depth = int(n).bit_length() - 1
            assert len(packed) == 32 + 64 * depth and packed[:4] == b"DPF2" and packed[4] == depth
            assert packed[5:16] == bytes(11) and packed[16:32] == k[129 * 4:130 * 4].tobytes()
            assert np.array_equal(b200dpf.key_unpack(packed), k)
    k = torch.from_numpy(golden["keys_a"][5].copy())
    assert torch.equal(dpf_cpp.key_unpack(dpf_cpp.key_pack(k)), k)
    with pytest.raises(b200dpf.B200DPFError, match="bad header"):
        b200dpf.key_unpack(b"XXXX" + bytes(100))
    good = b200dpf.key_pack(golden["keys_a"][5])
    with pytest.raises(b200dpf.B200DPFError, match="does not match"):
        b200dpf.key_unpack(good[:-1])
    with pytest.raises(b200dpf.B200DPFError, match="malformed"):
        b200dpf.key_pack(np.zeros(524, np.int32))


def test_non_power_of_two_domains_opt_in():
    import dpf
    d = dpf.DPF(prf=dpf.DPF.PRF_CHACHA20, allow_non_pow2=True)
    n = 1000
    table = torch.arange(n * 3, dtype=torch.int32).reshape(n, 3)
    k1, k2 = d.gen(999, n)
    assert int(k1.view(torch.int32)[130 * 4]) == 1024          # keys live in the padded domain
    d.table = dpf._pad_rows_to_pow2(table)                      # what eval_init stores (no GPU needed here)
    rec = d.eval_cpu([k1]) - d.eval_cpu([k2])
    assert torch.equal(rec[0], table[999])
    with pytest.raises(Exception, match="must be less than n"):
        d.gen(1000, n)
    with pytest.raises(Exception, match="power of two"):
        dpf.DPF().gen(5, n)                                     # default: the reference's behaviour


def test_python_gen_is_reference_compatible(golden):
    """dpf_cpp.gen(k, n, seed, prf) with the same first 4 seed bytes reproduces the
    reference's keys bit for bit (dpf_wrapper.cu:52 seeds mt19937 from them)."""
    import dpf_cpp
    for ci in (0, 9, 18, 27):
        prf, n, alpha, seed32 = [int(v) for v in golden["case_meta"][ci]]
        seed = seed32.to_bytes(4, "little") + b"\x00" * 124
        k1, k2 = dpf_cpp.gen(alpha, n, seed, prf)
        assert np.array_equal(k1.numpy(), golden["keys_a"][ci])
        assert np.array_equal(k2.numpy(), golden["keys_b"][ci])


def test_gpu_entry_points_fail_loudly_without_a_gpu():
    """No CUDA device in this container: every GPU entry point returns B200DPF_ECUDA with a message that says
    so -- there is no CPU evaluation behind the product API."""
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible here")
    L = b200dpf.lib()
    table = np.arange(256 * 16, dtype=np.int32).reshape(256, 16)
    h = C.c_void_p()
    ptr = table.ctypes.data_as(C.c_void_p)
    assert L.b200dpf_create(C.byref(h), ptr, 256, 16, 0, 0, 1) == -2 and b"no CUDA device" in L.b200dpf_last_error()
    devs = (C.c_int * 2)(0, 1)
    assert L.b200dpf_create_multi(C.byref(h), ptr, 256, 16, devs, 2, 0) == -2 and b"no CUDA device" in L.b200dpf_last_error()
    tabs = (C.c_void_p * 1)(table.ctypes.data)
    sizes = np.array([256], np.int64)
    assert L.b200dpf_group_create(C.byref(h), tabs, sizes, 1, 16, 0) == -2 and b"no CUDA device" in L.b200dpf_last_error()
    with pytest.raises(b200dpf.B200DPFError, match="no CUDA device"):
        b200dpf.gen_batch_gpu([1, 2], 256, bytes(88), 3)
    a, b = b200dpf.gen_batch_secure([1, 2], 256, bytes(88), 3)          # the CPU keygen is its own API, not a fallback
    assert a.shape == (2, 524)


def test_sharded_key_validation_without_a_gpu():
    """ShardedDPF refuses keys made for another table size before anything reaches a GPU (the device-resident
    path takes the tree depth from the context, so a wrong key would otherwise evaluate to garbage)."""
    from sharded import ShardedDPF, key_slice
    d = ShardedDPF(prf=2)
    d.n, d.entry_size = 1024, 16
    good, _ = b200dpf.gen(5, 1024, 1, 2)
    wrong, _ = b200dpf.gen(5, 2048, 1, 2)
    d._check_keys(torch.from_numpy(np.stack([good, good])))
    with pytest.raises(RuntimeError, match="different table size"):
        d._check_keys(torch.from_numpy(np.stack([good, wrong])))
    with pytest.raises(Exception, match=r"int32 \[B, 524\]"):
        d._check_keys(torch.zeros((2, 100), dtype=torch.int32))
    assert [key_slice(70, r, 3) for r in range(3)] == [(0, 24), (24, 48), (48, 70)]


def test_binned_dpf_argument_checks_without_a_gpu():
    import dpf
    d = dpf.BinnedDPF(prf=dpf.DPF.PRF_SALSA20)
    with pytest.raises(Exception, match="power of two"):
        d.eval_init([torch.zeros((100, 16), dtype=torch.int32)])
    with pytest.raises(Exception, match="eval_init"):
        d.eval_gpu([], [])
    assert "uninitialized" in repr(d)
