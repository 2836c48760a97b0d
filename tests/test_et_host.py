"""Early-terminated keys (four table rows per GGM leaf) on the host: key generation, the CPU
evaluation, the compact form, the argument checks and the Python CPU paths.  No GPU needed."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402
import et_oracle  # noqa: E402
import oracle  # noqa: E402

PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
EINVAL, ECUDA = -1, -2


@pytest.fixture(scope="module")
def orc():
    return oracle.Oracle()


def seed44(i):
    return bytes((31 * i + 7 * k + 1) & 0xFF for k in range(44))


def reconstruct(a, b, prf, orc):
    ra = et_oracle.eval_full_flat_et(orc, a, prf).view(np.uint32)
    rb = et_oracle.eval_full_flat_et(orc, b, prf).view(np.uint32)
    return ra - rb


def alphas_for(n):
    if n <= 64:
        return list(range(n))
    return sorted({0, 1, 2, 3, n // 2 + 1, n // 2 + 2, n - 2, n - 1})


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("n", [8, 16, 64, 1024, 1 << 14])
def test_oracle_reconstructs_one_hot(prf, n, orc):
    for i, alpha in enumerate(alphas_for(n)):
        a, b = B.gen_et(alpha, n, seed44(i), prf)
        d = reconstruct(a, b, prf, orc)
        exp = np.zeros(n, np.uint32)
        exp[alpha] = 1
        assert np.array_equal(d, exp), (prf, n, alpha)


@pytest.mark.parametrize("prf", PRFS)
def test_host_eval_reconstructs_every_alpha_small_n(prf):
    for n in (8, 32, 256, 1024):
        for alpha in range(n):
            a, b = B.gen_et(alpha, n, seed44(alpha), prf)
            d = B.eval_cpu_et(a, prf).view(np.uint32) - B.eval_cpu_et(b, prf).view(np.uint32)
            assert d[alpha] == 1 and np.count_nonzero(d) == 1, (prf, n, alpha)


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("n", [8, 16, 128, 1024, 1 << 12])
def test_host_eval_matches_oracle(prf, n, orc):
    for i, alpha in enumerate((0, n - 1, 5 % n, n // 2 + 3)):
        a, b = B.gen_et(alpha, n, seed44(100 + i), prf)
        for k in (a, b):
            assert np.array_equal(B.eval_cpu_et(k, prf), et_oracle.eval_full_flat_et(orc, k, prf))


def test_host_eval_matches_oracle_large(orc):
    n = 1 << 16
    a, _ = B.gen_et(40001, n, seed44(9), B.PRF_AES128)
    assert np.array_equal(B.eval_cpu_et(a, B.PRF_AES128), et_oracle.eval_full_flat_et(orc, a, B.PRF_AES128))


def test_key_layout():
    a, b = B.gen_et(77, 1 << 10, seed44(1), B.PRF_AES128)
    for k in (a, b):
        assert list(k[:4]) == [8, 2, 0, 0]                 # d = log2(n) - 2, word 1 = log2 rows per leaf
        assert list(k[520:524]) == [1024, 0, 0, 0]         # slot 130 = n rows
        assert not k[4 + 4 * 2 * 8:4 + 4 * 64].any()       # cw_1 beyond level d-1 is zero
    assert B.lib().b200dpf_ctx_rows_per_leaf(None) == -1


def test_determinism_and_batch():
    n, prf = 1 << 12, B.PRF_CHACHA20
    alphas = np.array([0, 1, 2, 3, 4095, 1234, 777, 2048, 5, 6, 7, 8], np.int64)
    seeds = b"".join(seed44(i) for i in range(len(alphas)))
    loop = [B.gen_et(int(al), n, seeds[44 * i:44 * i + 44], prf) for i, al in enumerate(alphas)]
    one_a, one_b = B.gen_batch_et(alphas, n, seeds, prf, nthreads=1)
    all_a, all_b = B.gen_batch_et(alphas, n, seeds, prf, nthreads=0)
    for i in range(len(alphas)):
        assert np.array_equal(one_a[i], loop[i][0]) and np.array_equal(one_b[i], loop[i][1])
    assert np.array_equal(one_a, all_a) and np.array_equal(one_b, all_b)
    again = B.gen_et(int(alphas[0]), n, seeds[:44], prf)
    assert np.array_equal(again[0], loop[0][0])


def test_golden_fixture():
    g = np.load(os.path.join(HERE, "golden", "et_v1.npz"))
    count = 0
    for prf in PRFS:
        for logn in (10, 14):
            tag = "p%d_n%d" % (prf, logn)
            n, alpha = 1 << logn, int(g[tag + "_alpha"])
            a, b = B.gen_et(alpha, n, g[tag + "_seed"].tobytes(), prf)
            assert np.array_equal(a, g[tag + "_key_a"]) and np.array_equal(b, g[tag + "_key_b"]), tag
            assert np.array_equal(B.eval_cpu_et(a, prf), g[tag + "_share_a"]), tag
            assert np.array_equal(B.eval_cpu_et(b, prf), g[tag + "_share_b"]), tag
            d = g[tag + "_share_a"].view(np.uint32) - g[tag + "_share_b"].view(np.uint32)
            assert d[alpha] == 1 and np.count_nonzero(d) == 1
            count += 1
    assert count == 8


def test_standard_entry_points_refuse_et_keys():
    L = B.lib()
    a, _ = B.gen_et(5, 1 << 10, seed44(2), B.PRF_AES128)
    out = np.zeros(1 << 10, np.int32)
    assert L.b200dpf_eval_cpu(a, B.PRF_AES128, out) == EINVAL
    assert L.b200dpf_key_n(a) == -1 and L.b200dpf_key_depth(a) == -1
    buf = C.create_string_buffer(L.b200dpf_key_packed_size(32))
    assert L.b200dpf_key_pack(a, buf, len(buf), None) == EINVAL
    packed = B.key_pack_et(a)
    assert packed[:4] == b"DPE4"
    assert L.b200dpf_key_unpack(packed, len(packed), np.zeros(524, np.int32)) == EINVAL


def test_et_entry_points_refuse_standard_keys():
    L = B.lib()
    s, _ = B.gen_secure(5, 1 << 10, seed44(3), B.PRF_AES128)
    assert L.b200dpf_eval_cpu_et(s, B.PRF_AES128, np.zeros(1 << 10, np.int32)) == EINVAL
    buf = C.create_string_buffer(L.b200dpf_key_packed_size(32))
    assert L.b200dpf_key_pack_et(s, buf, len(buf), None) == EINVAL
    packed = B.key_pack(s)
    assert L.b200dpf_key_unpack_et(packed, len(packed), np.zeros(524, np.int32)) == EINVAL


def test_argument_checks():
    L = B.lib()
    a, b = np.zeros(524, np.int32), np.zeros(524, np.int32)
    seed = seed44(4)
    for alpha, n in ((0, 12), (0, 4), (0, 2), (0, 1 << 32), (8, 8), (-1, 8)):
        assert L.b200dpf_gen_et(alpha, n, seed, 44, B.PRF_AES128, a, b) == EINVAL, (alpha, n)
    assert L.b200dpf_gen_et(0, 1 << 31, seed, 44, 7, a, b) == EINVAL
    assert L.b200dpf_gen_et(0, 16, seed, 43, B.PRF_AES128, a, b) == EINVAL
    assert L.b200dpf_gen_et(0, 16, None, 0, B.PRF_AES128, a, b) == EINVAL
    assert L.b200dpf_gen_et(0, 8, seed, 44, B.PRF_AES128, a, b) == 0
    assert L.b200dpf_eval_cpu_et(a, 9, np.zeros(8, np.int32)) == EINVAL
    table = np.zeros((64, 4), np.int32)
    h = C.c_void_p()
    rc = L.b200dpf_create_et(C.byref(h), table.ctypes.data_as(C.c_void_p), 64, 4, 0, 0, 1)
    assert rc in (0, ECUDA)
    if rc == 0:             # a machine with a GPU: the shape checks still apply
        L.b200dpf_destroy(h)
    else:
        assert b"no CUDA device" in L.b200dpf_last_error()
    for n, g in ((4, 1), (48, 1), (64, 16)):
        assert L.b200dpf_create_et(C.byref(h), table.ctypes.data_as(C.c_void_p), n, 4, 0, 0, g) == EINVAL, (n, g)


def test_compact_round_trip():
    for logn in (3, 10, 20):
        a, _ = B.gen_et(5, 1 << logn, seed44(5), B.PRF_SALSA20)
        packed = B.key_pack_et(a)
        assert len(packed) == 32 + 64 * (logn - 2)
        assert np.array_equal(B.key_unpack_et(packed), a)
    bad = bytearray(packed)
    bad[4] += 1
    with pytest.raises(B.B200DPFError):
        B.key_unpack_et(bytes(bad))


def test_python_cpu_paths():
    torch = pytest.importorskip("torch")
    import dpf
    d = dpf.DPF(prf=dpf.DPF.PRF_CHACHA20, early_termination=True)
    n = 256
    table = torch.randint(-2**31, 2**31 - 1, (n, 5), dtype=torch.int64).to(torch.int32)
    d.table = table
    for k in (0, 3, 130, 255):
        ka, kb = d.gen(k, n, seed=seed44(k))
        ra, rb = d.eval_cpu([ka]), d.eval_cpu([kb])
        assert torch.equal((ra - rb).to(torch.int32)[0], table[k])
    ka, kb = d.gen(7, n)                                # fresh os.urandom seed
    diff = d.eval_cpu([ka], one_hot_only=True) - d.eval_cpu([kb], one_hot_only=True)
    assert int(diff[0, 7]) == 1 and int(diff.abs().sum()) == 1
    a, b = d.gen_batch([1, 2, 3], n, seeds=b"".join(seed44(i) for i in range(3)))
    assert a.shape == (3, 524) and torch.equal(a[1], d.gen(2, n, seed=seed44(1))[0])
    with pytest.raises(Exception):
        d.gen(1, n, seed=b"short")
    with pytest.raises(Exception):
        d.gen(1, n, seed=seed44(1), secure=False)
    with pytest.raises(Exception):
        d.gen_batch([1, 2], n, seeds=[1, 2])
    with pytest.raises(Exception):
        dpf.DPF(devices=[0, 1], early_termination=True)
    with pytest.raises(Exception):
        dpf.BinnedDPF(early_termination=True)
    import sharded
    with pytest.raises(Exception):
        sharded.ShardedDPF(early_termination=True)
