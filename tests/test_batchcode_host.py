"""Batch codes on the host (include/b200dpf.h, b200dpf_batchcode_*): the layout's permutations against a restatement
written from the header, the copies' placement, the client's plan against a restatement of the same Kuhn order and
against scipy's maximum matching, an end-to-end retrieval from CPU share vectors for every kind of key, and the
refusals.  No GPU needed."""
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
from batchcode_ref import locate, per_copy, perm  # noqa: E402  (the layout, restated from include/b200dpf.h)

EINVAL, ECUDA, ESTATE = -1, -2, -4
M64 = (1 << 64) - 1
SEEDS = (0, 1, 0x0123456789ABCDEF, M64)


# ---- the plan, restated: Kuhn's augmenting paths, rows in order, copies 0, 1, 2 ------------------------------------

def plan_ref(n, nbins, seed, wanted):
    wanted = [int(r) for r in wanted]
    distinct = sorted(set(wanted))
    bins_of = {}
    for c in range(3):
        for r, b in zip(distinct, perm(n, seed, c, distinct) % nbins):
            bins_of.setdefault(r, []).append(int(b))
    match = {}                      # bin -> (wanted index, copy)
    first = {}
    for i, r in enumerate(wanted):
        if r in first:
            continue
        first[r] = i
        visited = set()

        def search(u):
            for c in range(3):
                v = bins_of[wanted[u]][c]
                if v in visited:
                    continue
                visited.add(v)
                if v not in match or search(match[v][0]):
                    match[v] = (u, c)
                    return True
            return False
        search(i)
    slot_of = {u: v for v, (u, _) in match.items()}
    slots = np.array([slot_of.get(first[r], -1) for r in wanted], np.int32)
    alphas = np.zeros(nbins, np.int64)
    for v, (u, c) in match.items():
        x = int(perm(n, seed, c, [wanted[u]])[0])
        alphas[v] = c * per_copy(n, nbins, v) + x // nbins
    return alphas, slots


@pytest.fixture(autouse=True)
def _deep_recursion():
    old = sys.getrecursionlimit()
    sys.setrecursionlimit(max(old, 20000))
    yield
    sys.setrecursionlimit(old)


# ---- tests ------------------------------------------------------------------------------------------------------

def test_symbols_present():
    L = C.CDLL(B.LIB_PATH)
    for name in ("b200dpf_batchcode_create", "b200dpf_batchcode_layout", "b200dpf_batchcode_locate", "b200dpf_batchcode_plan",
                 "b200dpf_batchcode_plan_device", "b200dpf_batchcode_update_rows"):
        assert name in B.SYMBOLS
        assert hasattr(L, name)


@pytest.mark.parametrize("n", [1, 2, 3, 7, 8, 9, 255, 256, 257, 1000, (1 << 16) + 1, 10 ** 6 + 3])
def test_permutations_are_bijections_equal_to_the_restatement(n):
    rng = np.random.RandomState(n % 1000)
    rows = np.arange(n)
    sample = rows if n <= 4096 else np.unique(np.concatenate([rng.randint(0, n, 1500), [0, 1, n - 2, n - 1]]))
    for seed in SEEDS:
        nbins = max(1, min(n, 7))
        for c in range(3):
            x = perm(n, seed, c, rows)
            assert np.array_equal(np.sort(x), rows), "pi_%d is not a bijection of [0, %d) (seed %x)" % (c, n, seed)
            for r in sample:       # the library's pi_c(r), read back from the copy's bin and in-bin row
                bins, in_bin = locate(n, nbins, seed, int(r))
                m = per_copy(n, nbins, bins[c])
                assert in_bin[c] // m == c
                assert (in_bin[c] - c * m) * nbins + bins[c] == x[r], (n, seed, c, r)


@pytest.mark.parametrize("n,nbins", [(1, 1), (2, 2), (3, 1), (9, 4), (257, 16), (1000, 1000), (1000, 3), (4099, 48),
                                     (20000, 1536)])
def test_locate_fills_every_bin_exactly(n, nbins):
    seed = 0xFEEDFACECAFEBEEF
    seen = [np.zeros(3 * per_copy(n, nbins, j), np.int32) for j in range(nbins)]
    for r in range(n):
        bins, rows = locate(n, nbins, seed, r)
        for c in range(3):
            assert 0 <= bins[c] < nbins and 0 <= rows[c] < 3 * per_copy(n, nbins, bins[c])
            seen[bins[c]][rows[c]] += 1
    for j in range(nbins):
        assert (seen[j] == 1).all(), "bin %d: rows not hit exactly once" % j
    assert sum(len(s) for s in seen) == 3 * n


def _check_matching(n, nbins, seed, wanted, alphas, slots):
    """valid (each slot one of its row's bins, distinct rows in distinct bins, alphas the copy's row) and maximum"""
    scipy_sparse = pytest.importorskip("scipy.sparse")
    from scipy.sparse.csgraph import maximum_bipartite_matching
    owner = {}
    for i, r in enumerate(wanted):
        s = int(slots[i])
        if s < 0:
            continue
        bins, rows = locate(n, nbins, seed, int(r))
        assert s in bins
        assert int(alphas[s]) in [rows[c] for c in range(3) if bins[c] == s]
        assert owner.setdefault(s, int(r)) == int(r), "bin %d answers two different rows" % s
    distinct = sorted(set(int(r) for r in wanted))
    edges = np.zeros((len(distinct), nbins), np.int8)
    for i, r in enumerate(distinct):
        for b in locate(n, nbins, seed, r)[0]:
            edges[i, b] = 1
    best = maximum_bipartite_matching(scipy_sparse.csr_matrix(edges), perm_type="column")
    assert len(owner) == int((best >= 0).sum())
    for j in set(range(nbins)) - set(owner):
        assert alphas[j] == 0


@pytest.mark.parametrize("n,nbins,k,dups", [
    (1, 1, 1, False), (1, 1, 3, True), (5, 1, 3, False), (7, 2, 5, True), (50, 7, 4, False), (1000, 16, 24, True),
    (4096, 48, 32, False), (10 ** 5, 300, 200, True), (10 ** 6 + 3, 2000, 1333, False), ((1 << 20) + 1, 2000, 2600, True),
    (3000, 12, 40, True),
])
def test_plan_equals_the_restated_kuhn_order_and_is_maximum(n, nbins, k, dups):
    rng = np.random.RandomState(n % 9973 + k)
    seed = int(rng.randint(0, 1 << 62))
    nq = 3 if k <= 200 else 1
    wanted = rng.randint(0, n, size=(nq, k)).astype(np.int64)
    if dups:
        wanted[:, k // 2:] = wanted[:, :k - k // 2][:, rng.permutation(k - k // 2)]
    alphas, slots = B.batchcode_plan(n, nbins, seed, wanted)
    assert alphas.shape == (nq, nbins) and slots.shape == (nq, k)
    for q in range(nq):
        ra, rs = plan_ref(n, nbins, seed, wanted[q])
        assert np.array_equal(slots[q], rs), "query %d: slots differ" % q
        assert np.array_equal(alphas[q], ra), "query %d: alphas differ" % q
        if nbins * k <= 300 * 200:
            _check_matching(n, nbins, seed, wanted[q], alphas[q], slots[q])


def test_plan_places_most_rows_at_one_and_a_half_bins_per_row():
    """k = 32 rows in 48 bins: well above the ~75 % that one copy per row in disjoint bins would reach"""
    rng = np.random.RandomState(5)
    n = 1 << 20
    wanted = np.stack([rng.choice(n, 32, replace=False) for _ in range(64)]).astype(np.int64)
    _, slots = B.batchcode_plan(n, 48, 99, wanted)
    assert (slots >= 0).mean() > 0.97


def _kind_args(kind):
    return {"": {}, "_et": {"early_termination": True}, "_xor": {"xor": True}}[kind]


@pytest.mark.parametrize("kind", ["", "_et", "_xor"])
def test_end_to_end_from_cpu_shares(kind):
    """bins built from locate, keys from BatchCodeDPF.gen_queries, answers from the CPU share vectors, reconstruct"""
    torch = pytest.importorskip("torch")
    import dpf
    n, nbins, k, E, nq = 301, 12, 8, 3, 2
    seed = 0xABCDEF
    rng = np.random.RandomState(7)
    table = rng.randint(-2 ** 31, 2 ** 31, size=(n, E), dtype=np.int64).astype(np.int32)
    d = dpf.BatchCodeDPF(dpf.DPF.PRF_CHACHA20, 0, nbins, seed=seed, **_kind_args(kind))
    d.use_layout(n)
    sizes = d.bin_sizes
    bins = [np.zeros((s, E), np.int32) for s in sizes]
    for r in range(n):
        bs, rows = locate(n, nbins, seed, r)
        for c in range(3):
            bins[bs[c]][rows[c]] = table[r]
    wanted = rng.randint(0, n, size=(nq, k)).astype(np.int64)
    wanted[1, 5] = wanted[1, 2]
    qa, qb, slots = d.gen_queries(torch.as_tensor(wanted))
    kid = B.KIND_IDS[kind]
    ev = {"": dpf.dpf_cpp.eval_cpu, "_et": dpf.dpf_cpp.eval_cpu_et, "_xor": dpf.dpf_cpp.eval_cpu_xor}[kind]

    def answer(key, g):
        share = ev(key, dpf.DPF.PRF_CHACHA20).numpy()
        if kind == "_xor":
            share = ((share.view(np.uint32)[:, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(-1)
        idx = [B.trimmed_alpha(r, sizes[g], kid) for r in range(sizes[g])]
        s = share[idx].astype(np.uint64)
        t = bins[g].view(np.uint32).astype(np.uint64)
        if kind == "_xor":
            return np.bitwise_xor.reduce(np.where(s[:, None] == 1, t, 0), axis=0).astype(np.uint32).view(np.int32)
        return ((s[:, None] * t).sum(axis=0) & 0xFFFFFFFF).astype(np.uint32).view(np.int32)

    out_a = torch.as_tensor(np.array([[answer(qa[q, g], g) for g in range(nbins)] for q in range(nq)]))
    out_b = torch.as_tensor(np.array([[answer(qb[q, g], g) for g in range(nbins)] for q in range(nq)]))
    rows, found = d.reconstruct(out_a, out_b, slots)
    assert found.numpy().mean() > 0.5
    for q in range(nq):
        for i in range(k):
            if found[q, i]:
                assert np.array_equal(rows[q, i].numpy(), table[wanted[q, i]]), (q, i)
            else:
                assert not rows[q, i].any()
    assert bool(found[1, 5]) == bool(found[1, 2]) and int(slots[1, 5]) == int(slots[1, 2])


def test_refusals():
    L = B.lib()
    b3, r3 = np.zeros(3, np.int32), np.zeros(3, np.int64)
    for n, nbins in ((0, 1), ((1 << 31) + 1, 8), (10, 0), (10, 11), ((1 << 22), (1 << 20) + 1), (1 << 31, 1), (1 << 31, 3)):
        assert L.b200dpf_batchcode_locate(n, nbins, 0, 0, b3, r3) == EINVAL, (n, nbins)
    assert L.b200dpf_batchcode_locate(1 << 31, 4, 0, 0, b3, r3) == 0         # 3 * 2^29 rows per bin fit
    assert L.b200dpf_batchcode_locate(10, 3, 0, 10, b3, r3) == EINVAL
    assert L.b200dpf_batchcode_locate(10, 3, 0, -1, b3, r3) == EINVAL
    assert "out of range" in L.b200dpf_last_error().decode()
    w = np.zeros((2, 4), np.int64)
    a, s = np.zeros((2, 3), np.int64), np.zeros((2, 4), np.int32)
    assert L.b200dpf_batchcode_plan(10, 3, 0, w, 2, 4, a, s) == 0
    for nq, k in ((0, 4), (2, 0), (2, 4097), ((1 << 24) // 3 + 1, 4)):
        assert L.b200dpf_batchcode_plan(10, 3, 0, w, nq, k, a, s) == EINVAL, (nq, k)
    w[1, 3] = 10
    assert L.b200dpf_batchcode_plan(10, 3, 0, w, 2, 4, a, s) == EINVAL
    assert "wanted row 10 out of range" in L.b200dpf_last_error().decode()
    w[1, 3] = -1
    assert L.b200dpf_batchcode_plan(10, 3, 0, w, 2, 4, a, s) == EINVAL
    # no context: every context entry point refuses it
    n_, nb_, sd_ = C.c_int64(), C.c_int(), C.c_uint64()
    assert L.b200dpf_batchcode_layout(None, C.byref(n_), C.byref(nb_), C.byref(sd_)) == ESTATE
    assert "not a batch-code context" in L.b200dpf_last_error().decode()
    assert L.b200dpf_batchcode_plan_device(None, C.c_void_p(16), 1, 1, C.c_void_p(16), C.c_void_p(16), None) == ESTATE
    assert L.b200dpf_batchcode_update_rows(None, np.zeros(1, np.int64), np.zeros(1, np.int32), 1) == ESTATE
    # create: the arguments are checked before any device is looked for
    h = C.c_void_p()
    t = np.zeros((8, 4), np.int32)
    assert L.b200dpf_batchcode_create(None, t.ctypes.data, 8, 4, 2, 0, 0, 0) == EINVAL
    assert L.b200dpf_batchcode_create(C.byref(h), None, 8, 4, 2, 0, 0, 0) == EINVAL
    assert L.b200dpf_batchcode_create(C.byref(h), t.ctypes.data, 8, 4, 9, 0, 0, 0) == EINVAL
    assert L.b200dpf_batchcode_create(C.byref(h), t.ctypes.data, 8, 0, 2, 0, 0, 0) == EINVAL
    assert L.b200dpf_batchcode_create(C.byref(h), t.ctypes.data, 8, 4, 2, 0, 0, 3) == EINVAL
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
    t = np.zeros((8, 4), np.int32)
    assert L.b200dpf_batchcode_create(C.byref(h), t.ctypes.data, 8, 4, 2, 0, 0, 0) == ECUDA
    assert "no CUDA device" in L.b200dpf_last_error().decode()
    assert not h.value


def test_python_refusals():
    torch = pytest.importorskip("torch")
    import dpf
    with pytest.raises(Exception, match="nbins >= 1"):
        dpf.BatchCodeDPF(dpf.DPF.PRF_AES128, 0, 0)
    with pytest.raises(Exception, match="xor=True and early_termination=True"):
        dpf.BatchCodeDPF(dpf.DPF.PRF_AES128, 0, 4, xor=True, early_termination=True)
    d = dpf.BatchCodeDPF(dpf.DPF.PRF_AES128, 0, 4, seed=1)
    with pytest.raises(Exception, match="must call `eval_init`"):
        d.plan([[1, 2]])
    with pytest.raises(Exception, match="must call `eval_init`"):
        d.gen_queries_device(torch.zeros((1, 2), dtype=torch.int64))
    d.use_layout(100)
    with pytest.raises(Exception, match="integer tensor"):
        d.plan(torch.zeros((1, 2)))
    with pytest.raises(RuntimeError, match="out of range"):
        d.plan([[1, 100]])
    with pytest.raises(Exception, match="seeds must be bytes"):
        d.gen_queries([[1, 2]], seeds=b"x")
    alphas, slots = d.plan([3, 3, 99])
    assert alphas.shape == (1, 4) and slots.shape == (1, 3) and int(slots[0, 0]) == int(slots[0, 1]) >= 0
    with pytest.raises(Exception, match="answers must be"):
        d.reconstruct(torch.zeros((1, 4, 2), dtype=torch.int32), torch.zeros((1, 4, 2), dtype=torch.int32), torch.zeros(3))
    d.buffers = []
    with pytest.raises(Exception, match="wanted_dev must be a contiguous int64"):
        d.gen_queries_device(torch.zeros((1, 2), dtype=torch.int64))
    with pytest.raises(RuntimeError, match="empty buffer list"):
        dpf.dpf_cpp.batchcode_plan_device(16, 1, 1, [], 16, 16, 0)
    ctx = B.BatchCodeContext.__new__(B.BatchCodeContext)    # a context that was never created
    ctx.handle = C.c_void_p()
    with pytest.raises(B.B200DPFError, match=r"b200dpf_batchcode_layout failed \(-4\).*not a batch-code context"):
        ctx.layout
    with pytest.raises(B.B200DPFError, match=r"b200dpf_batchcode_plan_device failed \(-4\)"):
        ctx.plan_device(16, 1, 1, 16, 16)
