"""XOR-shared keys (128 table rows per GGM leaf, XOR results) on the host: key generation, the CPU
evaluation, the compact form, the refusals between key kinds, the argument checks and the Python CPU
paths.  No GPU needed."""
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
import oracle  # noqa: E402
import xor_oracle  # noqa: E402

PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
EINVAL, ECUDA = -1, -2


@pytest.fixture(scope="module")
def orc():
    return oracle.Oracle()


def seed44(i):
    return bytes((29 * i + 5 * k + 3) & 0xFF for k in range(44))


def one_hot(n, alpha):
    e = np.zeros(n, np.uint8)
    e[alpha] = 1
    return e


# every lane position class: the ends of each 32-bit word of a leaf, and both ends of the domain
LANE_ALPHAS = (0, 1, 31, 32, 63, 64, 95, 96, 127, 128, 255)


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("n", [256, 512, 1 << 12])
def test_oracle_reconstructs_one_hot(prf, n, orc):
    for i, alpha in enumerate(sorted({a % n for a in LANE_ALPHAS} | {n - 1, n - 128, n // 2 + 31})):
        a, b = B.gen_xor(alpha, n, seed44(i), prf)
        bits = xor_oracle.share_bits(orc, a, prf) ^ xor_oracle.share_bits(orc, b, prf)
        assert np.array_equal(bits, one_hot(n, alpha)), (prf, n, alpha)


@pytest.mark.parametrize("prf", PRFS)
def test_host_eval_reconstructs_every_lane(prf):
    n = 512
    for alpha in range(n):
        a, b = B.gen_xor(alpha, n, seed44(alpha), prf)
        d = xor_oracle.unpack_bits(B.eval_cpu_xor(a, prf) ^ B.eval_cpu_xor(b, prf))
        assert np.array_equal(d, one_hot(n, alpha)), (prf, alpha)


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("n", [256, 1024, 1 << 13])
def test_host_eval_matches_oracle(prf, n, orc):
    for i, alpha in enumerate((0, 31, 32, 127, n - 1, n // 2 + 3)):
        a, b = B.gen_xor(alpha, n, seed44(100 + i), prf)
        for k in (a, b):
            assert np.array_equal(B.eval_cpu_xor(k, prf), xor_oracle.pack_bits(xor_oracle.share_bits(orc, k, prf)))


def test_host_eval_matches_oracle_large(orc):
    n = 1 << 18
    a, b = B.gen_xor(200001, n, seed44(9), B.PRF_AES128)
    got = B.eval_cpu_xor(a, B.PRF_AES128)
    assert np.array_equal(got, xor_oracle.pack_bits(xor_oracle.share_bits(orc, a, B.PRF_AES128)))
    d = xor_oracle.unpack_bits(got ^ B.eval_cpu_xor(b, B.PRF_AES128))
    assert np.flatnonzero(d).tolist() == [200001]


@pytest.mark.parametrize("logn", range(8, 32))
def test_keygen_every_depth(logn, orc):
    """n = 2^8 .. 2^31 (tree depth 1 .. 24): layout, and the leaf of alpha and one other leaf per the oracle"""
    n = 1 << logn
    alpha = (0x9E3779B97F4A7C15 * logn) % n
    prf = PRFS[logn % 4]
    a, b = B.gen_xor(alpha, n, seed44(logn), prf)
    d = logn - 7
    for k in (a, b):
        assert list(k[:4]) == [d, 7, 0, 0]
        assert int(np.uint32(k[520])) == n and not k[521:524].any()
        assert not k[4 + 4 * 2 * d:4 * 65].any()              # cw_1 beyond level d-1 is zero
        assert B._key_n(k, "_xor") == n
    leaf = alpha >> 7
    va, vb = xor_oracle.leaf_value(orc, a, leaf, prf), xor_oracle.leaf_value(orc, b, leaf, prf)
    assert va ^ vb == 1 << (alpha & 127)
    other = leaf ^ ((1 << d) - 1) if d > 0 else leaf
    if other != leaf:
        assert xor_oracle.leaf_value(orc, a, other, prf) == xor_oracle.leaf_value(orc, b, other, prf)


def test_determinism_and_batch():
    n, prf = 1 << 12, B.PRF_CHACHA20
    alphas = np.array([0, 1, 31, 32, 127, 128, 4095, 1234, 777, 2048, 5, 6], np.int64)
    seeds = b"".join(seed44(i) for i in range(len(alphas)))
    loop = [B.gen_xor(int(al), n, seeds[44 * i:44 * i + 44], prf) for i, al in enumerate(alphas)]
    for nthreads in (1, 3, 0):
        ka, kb = B.gen_batch_xor(alphas, n, seeds, prf, nthreads=nthreads)
        for i in range(len(alphas)):
            assert np.array_equal(ka[i], loop[i][0]) and np.array_equal(kb[i], loop[i][1]), (nthreads, i)
    again = B.gen_xor(int(alphas[0]), n, seeds[:44], prf)
    assert np.array_equal(again[0], loop[0][0]) and np.array_equal(again[1], loop[0][1])
    other = B.gen_xor(int(alphas[0]), n, seed44(99), prf)
    assert not np.array_equal(other[0], loop[0][0])


def test_golden_fixture():
    g = np.load(os.path.join(HERE, "golden", "xor_v1.npz"))
    count = 0
    for prf in PRFS:
        for logn in (10, 14):
            tag = "p%d_n%d" % (prf, logn)
            n, alpha = 1 << logn, int(g[tag + "_alpha"])
            a, b = B.gen_xor(alpha, n, g[tag + "_seed"].tobytes(), prf)
            assert np.array_equal(a, g[tag + "_key_a"]) and np.array_equal(b, g[tag + "_key_b"]), tag
            assert np.array_equal(B.eval_cpu_xor(a, prf), g[tag + "_bits_a"]), tag
            assert np.array_equal(B.eval_cpu_xor(b, prf), g[tag + "_bits_b"]), tag
            d = xor_oracle.unpack_bits(g[tag + "_bits_a"] ^ g[tag + "_bits_b"])
            assert np.array_equal(d, one_hot(n, alpha)), tag
            count += 1
    assert count == 8


def _keys_of_every_kind(n=1 << 10, alpha=5):
    std, _ = B.gen_secure(alpha, n, seed44(2), B.PRF_AES128)
    et, _ = B.gen_et(alpha, n, seed44(2), B.PRF_AES128)
    xk, _ = B.gen_xor(alpha, n, seed44(2), B.PRF_AES128)
    return std, et, xk


def test_refusals_between_key_kinds():
    L = B.lib()
    n = 1 << 10
    std, et, xk = _keys_of_every_kind(n)
    buf = C.create_string_buffer(L.b200dpf_key_packed_size(32))
    zkey = np.zeros(524, np.int32)
    # XOR keys at the standard and early-terminated entry points
    assert L.b200dpf_key_n(xk) == -1 and L.b200dpf_key_depth(xk) == -1
    assert L.b200dpf_eval_cpu(xk, B.PRF_AES128, np.zeros(n, np.int32)) == EINVAL
    assert L.b200dpf_eval_cpu_et(xk, B.PRF_AES128, np.zeros(n, np.int32)) == EINVAL
    assert L.b200dpf_key_pack(xk, buf, len(buf), None) == EINVAL
    assert L.b200dpf_key_pack_et(xk, buf, len(buf), None) == EINVAL
    packed_x = B.key_pack_xor(xk)
    assert packed_x[:4] == b"DPX7"
    assert L.b200dpf_key_unpack(packed_x, len(packed_x), zkey) == EINVAL
    assert L.b200dpf_key_unpack_et(packed_x, len(packed_x), zkey) == EINVAL
    # standard and early-terminated keys at the XOR entry points
    for k, pack in ((std, B.key_pack), (et, B.key_pack_et)):
        assert L.b200dpf_eval_cpu_xor(k, B.PRF_AES128, np.zeros(n // 32, np.uint32)) == EINVAL
        assert L.b200dpf_key_pack_xor(k, buf, len(buf), None) == EINVAL
        p = pack(k)
        assert L.b200dpf_key_unpack_xor(p, len(p), zkey) == EINVAL
    with pytest.raises(B.B200DPFError):
        B.eval_cpu_xor(std, B.PRF_AES128)
    with pytest.raises(B.B200DPFError):
        B.eval_cpu_et(xk, B.PRF_AES128)


@pytest.mark.parametrize("key_kind", ["", "_et", "_xor"])
@pytest.mark.parametrize("entry_kind", ["", "_et", "_xor"])
def test_each_entry_point_takes_exactly_its_kind(key_kind, entry_kind):
    """eval_cpu*, key_pack* and key_unpack* accept keys of their own kind and refuse every other kind with
    EINVAL; b200dpf_key_n / _key_depth see only standard keys."""
    L = B.lib()
    n = 1 << 10
    key = dict(zip(("", "_et", "_xor"), _keys_of_every_kind(n)))[key_kind]
    packed = getattr(B, "key_pack" + key_kind)(key)
    want = 0 if key_kind == entry_kind else EINVAL
    out = np.zeros(n // 32, np.uint32) if entry_kind == "_xor" else np.zeros(n, np.int32)
    assert getattr(L, "b200dpf_eval_cpu" + entry_kind)(key, B.PRF_AES128, out) == want
    buf = C.create_string_buffer(L.b200dpf_key_packed_size(32))
    assert getattr(L, "b200dpf_key_pack" + entry_kind)(key, buf, len(buf), None) == want
    unpacked = np.zeros(524, np.int32)
    assert getattr(L, "b200dpf_key_unpack" + entry_kind)(packed, len(packed), unpacked) == want
    if want == 0:
        assert np.array_equal(unpacked, key)
    depth = 10 - B.KINDS[key_kind][0]
    assert L.b200dpf_key_n(key) == (n if key_kind == "" else -1)
    assert L.b200dpf_key_depth(key) == (depth if key_kind == "" else -1)


def test_argument_checks():
    L = B.lib()
    a, b = np.zeros(524, np.int32), np.zeros(524, np.int32)
    seed = seed44(4)
    for alpha, n in ((0, 128), (0, 8), (0, 384), (0, 1 << 32), (256, 256), (-1, 256)):
        assert L.b200dpf_gen_xor(alpha, n, seed, 44, B.PRF_AES128, a, b) == EINVAL, (alpha, n)
    assert L.b200dpf_gen_xor(0, 1 << 31, seed, 44, 7, a, b) == EINVAL
    assert L.b200dpf_gen_xor(0, 256, seed, 43, B.PRF_AES128, a, b) == EINVAL
    assert L.b200dpf_gen_xor(0, 256, None, 0, B.PRF_AES128, a, b) == EINVAL
    assert L.b200dpf_gen_xor(255, 256, seed, 44, B.PRF_AES128, a, b) == 0
    assert L.b200dpf_eval_cpu_xor(a, 9, np.zeros(8, np.uint32)) == EINVAL
    alphas = np.array([0, 300], np.int64)
    ka, kb = np.zeros((2, 524), np.int32), np.zeros((2, 524), np.int32)
    assert L.b200dpf_gen_batch_xor(alphas, seed * 2, 2, 256, B.PRF_AES128, 0, ka, kb) == EINVAL   # 300 >= n
    assert L.b200dpf_gen_batch_xor(alphas, None, 2, 512, B.PRF_AES128, 0, ka, kb) == EINVAL
    assert L.b200dpf_gen_batch_xor(alphas, seed * 2, 2, 512, B.PRF_AES128, 0, ka, kb) == 0


def test_create_xor_argument_checks():
    L = B.lib()
    table = np.zeros((1024, 4), np.int32)
    h = C.c_void_p()
    rc = L.b200dpf_create_xor(C.byref(h), table.ctypes.data_as(C.c_void_p), 256, 4, 0, 0, 1)
    assert rc in (0, ECUDA)
    if rc == 0:             # a machine with a GPU: the shape checks below still apply
        assert L.b200dpf_ctx_rows_per_leaf(h) == 128
        L.b200dpf_destroy(h)
    else:
        assert b"no CUDA device" in L.b200dpf_last_error()
    for n, e, g in ((128, 4, 1), (8, 4, 1), (384, 4, 1), (1 << 32, 4, 1), (1024, 4, 8), (1024, 4, 3),
                    (256, 4, 2), (256, 0, 1), (256, 4097, 1)):
        assert L.b200dpf_create_xor(C.byref(h), table.ctypes.data_as(C.c_void_p), n, e, 0, 0, g) == EINVAL, (n, e, g)
    assert L.b200dpf_create_xor(C.byref(h), None, 256, 4, 0, 0, 1) == EINVAL
    assert L.b200dpf_create_xor(None, table.ctypes.data_as(C.c_void_p), 256, 4, 0, 0, 1) == EINVAL
    with pytest.raises(ValueError):
        B.Context(table, xor=True, early_termination=True)


def test_compact_round_trip():
    for logn in (8, 10, 20, 31):
        a, _ = B.gen_xor(5, 1 << logn, seed44(5), B.PRF_SALSA20)
        packed = B.key_pack_xor(a)
        assert len(packed) == 32 + 64 * (logn - 7)
        assert packed[:4] == b"DPX7" and packed[4] == logn - 7
        assert np.array_equal(B.key_unpack_xor(packed), a)
    bad = bytearray(packed)
    bad[4] += 1
    with pytest.raises(B.B200DPFError):
        B.key_unpack_xor(bytes(bad))
    with pytest.raises(B.B200DPFError):
        B.key_unpack_xor(bytes(packed)[:-1])


def test_python_cpu_paths():
    torch = pytest.importorskip("torch")
    import dpf
    d = dpf.DPF(prf=dpf.DPF.PRF_CHACHA20, xor=True)
    n = 512
    table = torch.randint(-2**31, 2**31 - 1, (n, 5), dtype=torch.int64).to(torch.int32)
    d.table = table
    for k in (0, 31, 32, 127, 128, 511):
        ka, kb = d.gen(k, n, seed=seed44(k))
        ra, rb = d.eval_cpu([ka]), d.eval_cpu([kb])
        assert torch.equal(torch.bitwise_xor(ra, rb)[0], table[k])
        bits_a = d.eval_cpu([ka], one_hot_only=True)
        assert bits_a.dtype == torch.int32 and bits_a.shape == (1, n) and int(bits_a.max()) <= 1
        ref = xor_oracle.xor_rows(bits_a.numpy().astype(np.uint8), table.numpy())
        assert np.array_equal(ra.numpy(), ref)
    ka, kb = d.gen(7, n)                                # fresh os.urandom seed
    diff = torch.bitwise_xor(d.eval_cpu([ka], one_hot_only=True), d.eval_cpu([kb], one_hot_only=True))
    assert int(diff[0, 7]) == 1 and int(diff.sum()) == 1
    a, b = d.gen_batch([1, 2, 3], n, seeds=b"".join(seed44(i) for i in range(3)))
    assert a.shape == (3, 524) and torch.equal(a[1], d.gen(2, n, seed=seed44(1))[0])
    assert len(d.pack_keys([a[0]])[0]) == 32 + 64 * 2
    with pytest.raises(Exception):
        d.gen(1, n, seed=b"short")
    with pytest.raises(Exception):
        d.gen(1, n, seed=seed44(1), secure=False)
    with pytest.raises(Exception):
        d.gen_batch([1, 2], n, seeds=[1, 2])
    with pytest.raises(Exception, match="one of them"):
        dpf.DPF(xor=True, early_termination=True)
    with pytest.raises(Exception, match="multi-device"):
        dpf.DPF(devices=[0, 1], xor=True)
    with pytest.raises(Exception):
        dpf.BinnedDPF(xor=True)
    import sharded
    with pytest.raises(Exception):
        sharded.ShardedDPF(xor=True)
    # callers that do not pass xor keep the standard kind
    assert dpf.DPF().xor is False
