"""Trimmed tables (any row count, include/b200dpf.h "Trimmed tables") on the host: the key domain and the row
numbering against a restatement, key generation through DPF(trim=True) reconstructing every row on the CPU,
argument checks, and the GPU entry points failing cleanly without a device.  No GPU needed."""
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

PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
EINVAL, ECUDA = -1, -2
KINDS = ("", "_et", "_xor")
LANE_BITS = {"": 0, "_et": 2, "_xor": 7}
N_MIN = {"": 2, "_et": 8, "_xor": 256}


def ref_domain(n, kind):
    """the next power of two >= n, at least the kind's smallest key"""
    return max(1 << (n - 1).bit_length(), N_MIN[kind])


def ref_alpha(row, n, kind):
    """bitrev_d(row >> b) << b | (row & (2^b - 1)), d = log2 domain - b"""
    b = LANE_BITS[kind]
    d = ref_domain(n, kind).bit_length() - 1 - b
    leaf = row >> b
    rev = int(format(leaf, "0%db" % d)[::-1], 2) if d else 0
    return (rev << b) | (row & ((1 << b) - 1))


def interesting_n(kind):
    ns = {1, 2, 3, 2 ** 31, 2 ** 31 - 1, N_MIN[kind] - 1, N_MIN[kind], N_MIN[kind] + 1}
    for k in range(1, 31):
        ns |= {2 ** k - 1, 2 ** k, 2 ** k + 1}
    return sorted(x for x in ns if 1 <= x <= 2 ** 31)


@pytest.mark.parametrize("kind", KINDS)
def test_domain_and_alpha_match_restatement(kind):
    for n in interesting_n(kind):
        assert B.trimmed_domain(n, kind) == ref_domain(n, kind), n
        rows = {0, n - 1, n // 2, min(n - 1, 5), min(n - 1, 128), max(0, n - 129)}
        for r in sorted(rows):
            assert B.trimmed_alpha(r, n, kind) == ref_alpha(r, n, kind), (n, r)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", [1, 3, 7, 9, 100, 257, 700, 3000, 4097])
def test_alpha_is_injective_into_domain(kind, n):
    got = [B.trimmed_alpha(r, n, kind) for r in range(n)]
    N = B.trimmed_domain(n, kind)
    assert len(set(got)) == n and min(got) >= 0 and max(got) < N


def test_argument_errors():
    L = B.lib()
    for n in (0, -1, 2 ** 31 + 1):
        assert L.b200dpf_trimmed_domain(n, 0) == -1
        assert L.b200dpf_trimmed_alpha(0, n, 0) == -1
    for kind in (-1, 3):
        assert L.b200dpf_trimmed_domain(5, kind) == -1
        assert L.b200dpf_trimmed_alpha(0, 5, kind) == -1
    assert L.b200dpf_trimmed_alpha(-1, 5, 0) == -1
    assert L.b200dpf_trimmed_alpha(5, 5, 0) == -1
    assert L.b200dpf_ctx_trimmed(None) == -1
    assert L.b200dpf_ctx_table_rows(None) == -1
    with pytest.raises(ValueError):
        B.trimmed_alpha(7, 7)
    with pytest.raises(ValueError):
        B.trimmed_domain(0)


def test_create_argument_errors_before_device():
    """bad arguments are EINVAL before any device is touched"""
    L = B.lib()
    h = C.c_void_p()
    table = np.zeros((5, 4), np.int32)
    ptr = table.ctypes.data_as(C.c_void_p)
    assert L.b200dpf_create_trimmed(C.byref(h), ptr, 0, 4, 0, 0) == EINVAL
    assert L.b200dpf_create_trimmed(C.byref(h), ptr, 2 ** 31 + 1, 4, 0, 0) == EINVAL
    assert L.b200dpf_create_trimmed(C.byref(h), ptr, 5, 0, 0, 0) == EINVAL
    assert L.b200dpf_create_trimmed(C.byref(h), ptr, 5, 4, 0, 3) == EINVAL
    assert L.b200dpf_create_trimmed(C.byref(h), None, 5, 4, 0, 0) == EINVAL
    assert not h.value
    ptrs = (C.c_void_p * 2)(table.ctypes.data, table.ctypes.data)
    for sizes in ([5, 0], [5, 2 ** 31 + 1]):
        assert L.b200dpf_group_create_trimmed(C.byref(h), ptrs, np.array(sizes, np.int64), 2, 4, 0, 0) == EINVAL
    assert L.b200dpf_group_create_trimmed(C.byref(h), ptrs, np.array([5, 3], np.int64), 2, 4, 0, 7) == EINVAL
    assert not h.value


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the behaviour without a CUDA device")
def test_gpu_entry_points_fail_cleanly_without_device():
    L = B.lib()
    h = C.c_void_p()
    table = np.zeros((5, 4), np.int32)
    assert L.b200dpf_create_trimmed(C.byref(h), table.ctypes.data_as(C.c_void_p), 5, 4, 0, 0) == ECUDA
    assert "no CUDA device" in L.b200dpf_last_error().decode()
    ptrs = (C.c_void_p * 1)(table.ctypes.data)
    assert L.b200dpf_group_create_trimmed(C.byref(h), ptrs, np.array([5], np.int64), 1, 4, 0, 2) == ECUDA
    assert not h.value


# ---- DPF(trim=True): keys reconstruct every row through the CPU evaluation --------------------------------

def _dpf():
    import dpf
    return dpf


def _table(n, e, seed):
    return np.random.RandomState(seed).randint(-2 ** 31, 2 ** 31, size=(n, e), dtype=np.int64).astype(np.int32)


@pytest.mark.parametrize("kind", ["standard", "et", "xor"])
@pytest.mark.parametrize("prf", PRFS)
def test_dpf_trim_keys_reconstruct_rows_on_cpu(kind, prf):
    import torch
    dpf = _dpf()
    n, e = {"standard": 37, "et": 45, "xor": 300}[kind], 3
    d = dpf.DPF(prf=prf, trim=True, early_termination=kind == "et", xor=kind == "xor")
    table = torch.from_numpy(_table(n, e, prf))
    d.table = table            # eval_cpu only: no device upload
    rows = sorted({0, 1, n // 2, n - 2, n - 1})
    pairs = [d.gen(r, n) for r in rows]
    a = d.eval_cpu([p[0] for p in pairs])
    b = d.eval_cpu([p[1] for p in pairs])
    rec = (a ^ b) if kind == "xor" else (a - b)
    assert torch.equal(rec.to(torch.int32), table[rows])
    # the share vectors in row order: one-hot at the row
    sa = d.eval_cpu([pairs[1][0]], one_hot_only=True)
    sb = d.eval_cpu([pairs[1][1]], one_hot_only=True)
    diff = (sa ^ sb) if kind == "xor" else (sa - sb)
    assert diff.shape == (1, n) and torch.nonzero(diff[0]).flatten().tolist() == [rows[1]]


@pytest.mark.parametrize("kind", ["standard", "et", "xor"])
def test_dpf_trim_gen_batch_maps_rows(kind):
    import torch
    dpf = _dpf()
    n = {"standard": 1000, "et": 1001, "xor": 1500}[kind]
    d = dpf.DPF(prf=B.PRF_CHACHA20, trim=True, early_termination=kind == "et", xor=kind == "xor")
    rows = [0, 7, n - 1, 513]
    suffix = {"standard": "", "et": "_et", "xor": "_xor"}[kind]
    alphas = np.array([B.trimmed_alpha(r, n, suffix) for r in rows], np.int64)
    if kind == "standard":      # explicit integer seeds: the reference's generator
        seeds = np.arange(11, 11 + len(rows), dtype=np.uint32)
        ka, kb = d.gen_batch(rows, n, seeds=seeds.astype(np.int64))
        want_a, want_b = B.gen_batch(alphas, B.trimmed_domain(n), seeds, B.PRF_CHACHA20)
    else:
        ka, kb = d.gen_batch(rows, n, seeds=bytes(range(44)) * len(rows))
        want_a, want_b = getattr(B, "gen_batch" + suffix)(alphas, B.trimmed_domain(n, suffix), bytes(range(44)) * len(rows),
                                                          B.PRF_CHACHA20)
    assert np.array_equal(ka.numpy(), want_a) and np.array_equal(kb.numpy(), want_b)
    d.table = torch.from_numpy(_table(n, 2, 5))
    rec = (d.eval_cpu(list(ka)) ^ d.eval_cpu(list(kb))) if kind == "xor" else (d.eval_cpu(list(ka)) - d.eval_cpu(list(kb)))
    assert torch.equal(rec.to(torch.int32), d.table[rows])


def test_dpf_trim_argument_errors():
    dpf = _dpf()
    with pytest.raises(Exception, match="multi-device"):
        dpf.DPF(trim=True, devices=[0, 1])
    with pytest.raises(Exception, match="sharded"):
        dpf.DPF(trim=True, shard=(0, 2))
    d = dpf.DPF(trim=True)
    with pytest.raises(Exception, match="selected row"):
        d.gen(5, 5)
    with pytest.raises(Exception, match="rows in"):
        d.gen_batch([0, 5], 5)
    with pytest.raises(Exception, match="eval_init"):
        d.eval_cpu([d.gen(0, 5)[0]])
    # the defaults are unchanged: a DPF without trim still refuses a non-power-of-two domain
    with pytest.raises(Exception, match="power of two"):
        dpf.DPF().gen(0, 5)
