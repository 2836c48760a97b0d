"""Keyword PIR on the host (include/b200dpf.h, b200dpf_kwpir_*): the hash against a restatement written from the header,
the placement rule restated in numpy (every item placed, every slot filled at most once, and the failure past the round
cap), an end-to-end retrieval from CPU share vectors for every kind of key, and the refusals.  No GPU needed."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402
import kwpir_ref as K  # noqa: E402

EINVAL, ECUDA, ESTATE, EFULL = -1, -2, -4, -5
M64 = (1 << 64) - 1
SEEDS = (0, 1, 0x0123456789ABCDEF, M64)


def test_symbols_present():
    L = C.CDLL(B.LIB_PATH)
    for name in ("b200dpf_kwpir_create", "b200dpf_kwpir_layout", "b200dpf_kwpir_build_stats", "b200dpf_kwpir_locate",
                 "b200dpf_kwpir_plan_device", "b200dpf_kwpir_update", "b200dpf_kwpir_tags"):
        assert name in B.SYMBOLS
        assert hasattr(L, name)


@pytest.mark.parametrize("m", [1, 2, 3, 1000, (1 << 20) + 7, (1 << 31) - 1, 1 << 31])
def test_locate_equals_the_restated_hash(m):
    rng = np.random.RandomState(m % 1000)
    kw = np.concatenate([np.array([0, 1, 2, M64 - 1, 1 << 63, (1 << 63) - 1], np.uint64),
                         rng.randint(0, 1 << 62, 2000, dtype=np.int64).astype(np.uint64) * np.uint64(3),
                         np.arange(500, dtype=np.uint64)])
    for seed in SEEDS:
        got = B.kwpir_locate(m, seed, kw)
        assert got.shape == (len(kw), 3)
        assert np.array_equal(got, K.rows3(kw, m, seed)), (m, seed)
        assert (got >= 0).all() and (got < m).all()


def _check_placement(kw, m, seed, owner):
    """every item in exactly one slot, each slot holding at most one item, and that slot one of the item's candidates"""
    full = owner[owner >= 0]
    assert np.array_equal(np.sort(full), np.arange(len(kw)))
    slots = np.nonzero(owner >= 0)[0]
    items = owner[slots]
    assert np.array_equal(slots % m, K.rows3(kw[items], m, seed)[np.arange(len(items)), slots // m])


@pytest.mark.parametrize("n,expansion", [(1, 1.3), (2, 1.0), (3, 1.0), (100, 1.3), (4097, 1.3), (4097, 1.15), (1 << 14, 1.3)])
def test_restated_placement_places_every_item_once(n, expansion):
    rng = np.random.RandomState(n)
    kw = np.unique(rng.randint(0, 1 << 62, n * 2, dtype=np.int64).astype(np.uint64))[:n]
    rng.shuffle(kw)
    m = K.default_m(n, expansion)
    seed = 0xC0FFEE + n
    rounds, owner = K.place(kw, m, seed)
    assert rounds is not None and 1 <= rounds <= K.MAX_ROUNDS
    _check_placement(kw, m, seed, owner)
    t = K.tags(kw, owner, m)
    assert (t != 0).sum() == n


def test_restated_placement_fails_past_the_round_cap():
    """n = 3m items need every slot, and with ~3m e^-3 slots that no keyword hashes to, no placement exists"""
    m = 1000
    kw = np.arange(3 * m, dtype=np.uint64) * np.uint64(0x9E3779B1)
    rounds, owner = K.place(kw, m, 7)
    assert rounds is None
    assert len(set((np.arange(3) * m + K.rows3(kw, m, 7)).reshape(-1).tolist())) < 3 * m, "some slot is no keyword's candidate"
    assert (owner >= 0).sum() < 3 * m


def _kind_args(kind):
    return {"": {}, "_et": {"early_termination": True}, "_xor": {"xor": True}}[kind]


@pytest.mark.parametrize("kind", ["", "_et", "_xor"])
def test_end_to_end_from_cpu_shares(kind):
    """bins built from the restated placement, keys from KeywordDPF.gen_queries, answers from the CPU share vectors"""
    torch = pytest.importorskip("torch")
    import dpf
    n, E = 300, 3
    seed = 0xABCDEF
    rng = np.random.RandomState(11)
    kw = np.unique(rng.randint(0, 1 << 62, 2 * n, dtype=np.int64).astype(np.uint64) * np.uint64(2))[:n]
    kw[0], kw[1] = 0, M64 - 1
    values = rng.randint(-2 ** 31, 2 ** 31, size=(n, E), dtype=np.int64).astype(np.int32)
    m = K.default_m(n)
    rounds, owner = K.place(kw, m, seed)
    assert rounds is not None
    bins = np.zeros((3, m, E + 2), np.int32)
    for s in np.nonzero(owner >= 0)[0]:
        i = owner[s]
        tag = (int(kw[i]) + 1) & M64
        bins[s // m, s % m, :E] = values[i]
        bins[s // m, s % m, E:] = np.array([tag & 0xFFFFFFFF, tag >> 32], np.uint32).view(np.int32)
    d = dpf.KeywordDPF(dpf.DPF.PRF_CHACHA20, 0, seed=seed, **_kind_args(kind))
    d.use_layout(n, m, seed)
    absent = np.array([1, 3, M64 - 2, (1 << 63) + 5], np.uint64)     # odd: never among the even keywords
    query = np.concatenate([kw[:6], absent, kw[-3:]])
    qa, qb = d.gen_queries(query)
    assert qa.shape == (len(query), 3, B.KEY_WORDS)
    kid = B.KIND_IDS[kind]
    ev = {"": dpf.dpf_cpp.eval_cpu, "_et": dpf.dpf_cpp.eval_cpu_et, "_xor": dpf.dpf_cpp.eval_cpu_xor}[kind]
    order = [B.trimmed_alpha(r, m, kid) for r in range(m)]

    def answer(key, g):
        share = ev(key, dpf.DPF.PRF_CHACHA20).numpy()
        if kind == "_xor":
            share = ((share.view(np.uint32)[:, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(-1)
        s = share[order].astype(np.uint64)
        t = bins[g].view(np.uint32).astype(np.uint64)
        if kind == "_xor":
            return np.bitwise_xor.reduce(np.where(s[:, None] == 1, t, 0), axis=0).astype(np.uint32).view(np.int32)
        return ((s[:, None] * t).sum(axis=0) & 0xFFFFFFFF).astype(np.uint32).view(np.int32)

    out_a = torch.as_tensor(np.array([[answer(qa[q, g], g) for g in range(3)] for q in range(len(query))]))
    out_b = torch.as_tensor(np.array([[answer(qb[q, g], g) for g in range(3)] for q in range(len(query))]))
    vals, found = d.reconstruct(out_a, out_b, query)
    where = {int(w): i for i, w in enumerate(kw)}
    for q, w in enumerate(query):
        if int(w) in where:
            assert found[q] and np.array_equal(vals[q].numpy(), values[where[int(w)]]), q
        else:
            assert not found[q] and not vals[q].any(), q


def test_refusals():
    L = B.lib()
    kw = np.array([5, 6], np.uint64)
    r3 = np.zeros((2, 3), np.int64)
    for m in (0, -1, (1 << 31) + 1):
        assert L.b200dpf_kwpir_locate(m, 0, kw, 2, r3) == EINVAL, m
    assert L.b200dpf_kwpir_locate(10, 0, kw, -1, r3) == EINVAL
    assert L.b200dpf_kwpir_locate(10, 0, np.array([5, M64], np.uint64), 2, r3) == EINVAL
    assert "reserved" in L.b200dpf_last_error().decode()
    raw = C.CDLL(B.LIB_PATH)         # null buffers: untyped pointers
    raw.b200dpf_kwpir_locate.argtypes = [C.c_int64, C.c_uint64, C.c_void_p, C.c_int64, C.c_void_p]
    assert raw.b200dpf_kwpir_locate(10, 0, None, 2, r3.ctypes.data) == EINVAL
    assert raw.b200dpf_kwpir_locate(10, 0, kw.ctypes.data, 2, None) == EINVAL
    assert raw.b200dpf_kwpir_locate(10, 0, None, 0, None) == 0
    # no context: every context entry point refuses it
    n_, m_, sd_, e_ = C.c_int64(), C.c_int64(), C.c_uint64(), C.c_int()
    assert L.b200dpf_kwpir_layout(None, C.byref(n_), C.byref(m_), C.byref(sd_), C.byref(e_)) == ESTATE
    assert "not a keyword-PIR context" in L.b200dpf_last_error().decode()
    rounds, ms = C.c_int(), C.c_double()
    assert L.b200dpf_kwpir_build_stats(None, C.byref(rounds), C.byref(ms)) == ESTATE
    assert L.b200dpf_kwpir_plan_device(None, C.c_void_p(16), 1, C.c_void_p(16), None) == ESTATE
    assert L.b200dpf_kwpir_update(None, kw, np.zeros(2, np.int32), 2) == ESTATE
    assert L.b200dpf_kwpir_tags(None, np.zeros(3, np.uint64)) == ESTATE
    # create: the arguments are checked before any device is looked for
    h = C.c_void_p()
    k8 = np.arange(8, dtype=np.uint64)
    v8 = np.zeros((8, 4), np.int32)
    kp, vp = k8.ctypes.data, v8.ctypes.data
    assert L.b200dpf_kwpir_create(None, kp, vp, 8, 4, 3, 0, 0, 0) == EINVAL
    for args in ((None, vp, 8, 4, 3), (kp, None, 8, 4, 3), (kp, vp, 0, 4, 3), (kp, vp, (1 << 30) + 1, 4, 1 << 29),
                 (kp, vp, 8, 0, 3), (kp, vp, 8, 4095, 3), (kp, vp, 8, 4, 2), (kp, vp, 8, 4, (1 << 31) + 1)):
        assert L.b200dpf_kwpir_create(C.byref(h), *args, 0, 0, 0) == EINVAL, args
        assert not h.value
    assert "out of range" in L.b200dpf_last_error().decode()
    assert L.b200dpf_kwpir_create(C.byref(h), kp, vp, 8, 4, 3, 0, 0, 3) == EINVAL     # unknown kind
    assert not h.value


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the behaviour without a CUDA device")
def test_create_fails_cleanly_without_device():
    L = B.lib()
    h = C.c_void_p()
    k8 = np.arange(8, dtype=np.uint64)
    v8 = np.zeros((8, 4), np.int32)
    assert L.b200dpf_kwpir_create(C.byref(h), k8.ctypes.data, v8.ctypes.data, 8, 4, 3, 0, 0, 0) == ECUDA
    assert "no CUDA device" in L.b200dpf_last_error().decode()
    assert not h.value


def test_python_refusals():
    torch = pytest.importorskip("torch")
    import dpf
    with pytest.raises(Exception, match="expansion >= 1"):
        dpf.KeywordDPF(dpf.DPF.PRF_AES128, 0, expansion=0.9)
    with pytest.raises(Exception, match="xor=True and early_termination=True"):
        dpf.KeywordDPF(dpf.DPF.PRF_AES128, 0, xor=True, early_termination=True)
    d = dpf.KeywordDPF(dpf.DPF.PRF_AES128, 0, seed=1)
    with pytest.raises(Exception, match="must call `eval_init`"):
        d.plan([1, 2])
    with pytest.raises(Exception, match="must call `eval_init`"):
        d.gen_queries_device(torch.zeros(2, dtype=torch.int64))
    with pytest.raises(Exception, match="Must call `eval_init` before `update`"):
        d.update([1], [[1]])
    d.use_layout(100, 40, 1)
    with pytest.raises(Exception, match="1-D integer"):
        d.plan(torch.zeros(2))
    with pytest.raises(Exception, match="1-D integer"):
        d.plan([[1, 2]])
    with pytest.raises(RuntimeError, match="reserved"):
        d.plan(np.array([M64], np.uint64))
    with pytest.raises(Exception, match="seeds must be bytes"):
        d.gen_queries([1, 2], seeds=b"x")
    rows = d.plan([1 << 63, 7, M64 - 1])
    assert rows.shape == (3, 3)
    assert np.array_equal(rows.numpy(), K.rows3(np.array([1 << 63, 7, M64 - 1], np.uint64), 40, 1))
    d.value_size = 2
    with pytest.raises(Exception, match="answers must be"):
        d.reconstruct(torch.zeros((1, 3, 3), dtype=torch.int32), torch.zeros((1, 3, 3), dtype=torch.int32), [1])
    d.buffers = []
    with pytest.raises(Exception, match="keywords_dev must be a contiguous int64"):
        d.gen_queries_device(torch.zeros(2, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="empty buffer list"):
        dpf.dpf_cpp.kwpir_plan_device(16, 1, [], 16, 0)
    d.buffers = None
    ctx = B.KeywordContext.__new__(B.KeywordContext)    # a context that was never created
    ctx.handle = C.c_void_p()
    with pytest.raises(B.B200DPFError, match=r"b200dpf_kwpir_layout failed \(-4\).*not a keyword-PIR context"):
        ctx.layout
    with pytest.raises(B.B200DPFError, match=r"b200dpf_kwpir_plan_device failed \(-4\)"):
        ctx.plan_device(16, 1, 16)
