"""Keyword PIR on the GPU (b200dpf_kwpir_*): the placement built on the device equals the numpy restatement of the
header's rule byte for byte (several sizes, keyword patterns and loads, and under concurrent builds), a build past the
round cap fails with EFULL and KeywordDPF retries the next seeds, every present keyword reconstructs its value and every
absent one is not found for every kind of key, PRF, entry size and query path, the device locator equals the host's,
and value updates are applied, refused and ordered as documented."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402
import kwpir_ref as K  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
EINVAL, ESTATE, EFULL = -1, -4, -5
M64 = (1 << 64) - 1
KINDS = {"standard": ({}, ""), "et": ({"early_termination": True}, "_et"), "xor": ({"xor": True}, "_xor")}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


def keywords_of(pattern, n, seed):
    rng = np.random.RandomState(seed)
    if pattern == "sequential":
        return np.arange(n, dtype=np.uint64)
    if pattern == "high":
        return np.uint64(M64 - 1) - np.arange(n, dtype=np.uint64) * np.uint64(3)
    kw = np.unique(rng.randint(0, 1 << 63, 2 * n + 8, dtype=np.int64).astype(np.uint64) * np.uint64(2))[:n]
    rng.shuffle(kw)
    return kw


def create(keywords, values, m, seed, kind="", device_inputs=False, torch=None):
    """a KeywordContext from host arrays or from CUDA tensors (read in place)"""
    if not device_inputs:
        return B.KeywordContext(keywords, values, m, seed, early_termination=kind == "_et", xor=kind == "_xor")
    kt = torch.as_tensor(np.ascontiguousarray(keywords, np.uint64).view(np.int64)).cuda()
    vt = torch.as_tensor(values).cuda()
    ctx = B.KeywordContext.__new__(B.KeywordContext)
    ctx.n, ctx.value_size = values.shape
    ctx.entry_size = ctx.value_size + 2
    ctx.kind = kind
    ctx._trimmed = True
    ctx.handle = C.c_void_p()
    B._check(B.lib().b200dpf_kwpir_create(C.byref(ctx.handle), C.c_void_p(kt.data_ptr()), C.c_void_p(vt.data_ptr()), ctx.n,
                                          ctx.value_size, m, seed, 0, B.KIND_IDS[kind]), "b200dpf_kwpir_create")
    return ctx


PLACEMENTS = [(n, pattern, expansion) for n in (1, 2, 3, 100, 4097, 1 << 16, (1 << 20) + 1)
              for pattern in ("random", "sequential", "high") for expansion in (1.3, 1.15)]


@pytest.mark.parametrize("n,pattern,expansion", PLACEMENTS)
def test_placement_equals_the_restatement(torch_cuda, n, pattern, expansion):
    kw = keywords_of(pattern, n, n)
    m = K.default_m(n, expansion)
    seed = 0x5EED0000 + n
    rounds, owner = K.place(kw, m, seed)
    assert rounds is not None
    kind = ("", "_et", "_xor")[PLACEMENTS.index((n, pattern, expansion)) % 3]
    values = random_table(n, 1, seed=n)
    ctx = create(kw, values, m, seed, kind, device_inputs=n % 2 == 1, torch=torch_cuda)
    try:
        assert ctx.layout == (n, m, seed, 1)
        assert ctx.bin_rows == [m] * 3
        assert np.array_equal(ctx.tags(), K.tags(kw, owner, m))
        assert ctx.build_stats[0] == rounds
    finally:
        ctx.close()


def test_builds_are_identical_under_concurrent_builds(torch_cuda):
    n = 100000
    kw = keywords_of("random", n, 77)
    values = random_table(n, 14, seed=3)
    m = K.default_m(n)
    rounds, owner = K.place(kw, m, 99)
    want = K.tags(kw, owner, m)
    got, errors = [], []

    def build(i):
        try:
            for r in range(2):
                ctx = create(kw, values, m, 99, ("", "_et", "_xor")[(i + r) % 3], device_inputs=(i + r) % 2 == 1, torch=torch_cuda)
                try:
                    got.append(ctx.tags())
                finally:
                    ctx.close()
        except Exception as e:       # reported below
            errors.append(repr(e))

    def other(i):
        try:
            for r in range(3):
                okw = keywords_of("random", 30000 + i, i)
                ctx = create(okw, random_table(len(okw), 16, seed=i), K.default_m(len(okw)), i + r)
                ctx.close()
        except Exception as e:
            errors.append(repr(e))

    threads = [threading.Thread(target=build, args=(i,)) for i in range(3)] + \
              [threading.Thread(target=other, args=(i,)) for i in range(3)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
        assert not t.is_alive(), "a build thread did not finish"
    assert not errors, errors
    assert len(got) == 6
    for t in got:
        assert np.array_equal(t, want)


def test_full_placement_fails_and_the_python_layer_retries(torch_cuda):
    import dpf
    L = B.lib()
    # n = 3m: the restatement leaves items homeless after the round cap, so the create fails and creates nothing
    m = 1000
    kw = np.arange(3 * m, dtype=np.uint64) * np.uint64(0x9E3779B1)
    assert K.place(kw, m, 7)[0] is None
    values = np.zeros((3 * m, 2), np.int32)
    h = C.c_void_p()
    assert L.b200dpf_kwpir_create(C.byref(h), kw.ctypes.data, values.ctypes.data, 3 * m, 2, m, 7, 0, 0) == EFULL
    assert "homeless" in L.b200dpf_last_error().decode()
    assert not h.value
    with pytest.raises(B.B200DPFError, match=r"failed \(-5\)"):
        B.KeywordContext(kw, values, m, 7)
    with pytest.raises(Exception, match="did not finish for seeds 7..14"):
        dpf.KeywordDPF(dpf.DPF.PRF_AES128, 0, seed=7, expansion=1.0).eval_init(kw, values)
    # near the load threshold: find a seed the restatement fails with and a later one (within 8) it places with
    n = 600
    kw = keywords_of("random", n, 3)
    d = dpf.KeywordDPF(dpf.DPF.PRF_AES128, 0, seed=0, expansion=1.075)
    m = K.default_m(n, 1.075)
    ok = [K.place(kw, m, s)[0] is not None for s in range(40)]
    start = next(s for s in range(32) if not ok[s] and any(ok[s + 1:s + 8]))
    d.seed = start
    d.eval_init(kw, random_table(n, 3, seed=1))
    try:
        assert d.seed == next(s for s in range(start, start + 8) if ok[s])
        assert d.m == m
        assert dpf.dpf_cpp.kwpir_layout(d.buffers) == (n, m, d.seed, 3)
    finally:
        d.close()


# (kind, prf, value size, n, inputs on the device)
RETRIEVAL = [(kind, prf, e, n, dev) for kind in KINDS for prf in (B.PRF_AES128, B.PRF_CHACHA20)
             for e, n, dev in ((1, 3000, False), (14, 20011, True), (16, 20011, False), (125, 5000, True), (4094, 300, False))
             if (e, n) != (4094, 300) or prf == B.PRF_CHACHA20] + \
            [("standard", B.PRF_SALSA20, 14, 4097, True), ("et", B.PRF_DUMMY, 16, 4097, False), ("xor", B.PRF_SALSA20, 5, 700, True)]


@pytest.mark.parametrize("kind,prf,e,n,dev", RETRIEVAL)
def test_present_keywords_reconstruct_and_absent_ones_are_not_found(torch_cuda, kind, prf, e, n, dev):
    torch = torch_cuda
    import dpf
    kw_args, _ = KINDS[kind]
    kw = keywords_of("random", n, n + e)        # even keywords: odd ones are absent
    values = random_table(n, e, seed=e)
    d = dpf.KeywordDPF(prf, 0, seed=1234 + e, **kw_args)
    if dev:
        d.eval_init(torch.as_tensor(kw.view(np.int64)).cuda(), torch.as_tensor(values).cuda())
    else:
        d.eval_init(kw, values)
    try:
        rng = np.random.RandomState(prf + e)
        present = kw[rng.choice(n, min(n, 40), replace=False)]
        absent = np.array([1, 3, (1 << 63) + 1, M64 - 2] + list(rng.randint(0, 1 << 62, 8).astype(np.uint64) * np.uint64(2) + np.uint64(1)),
                          np.uint64)
        query = np.concatenate([present[:20], absent, present[20:]])
        qd = torch.as_tensor(query.view(np.int64)).cuda()
        runs = [d.gen_queries_device(qd, compact=True), d.gen_queries_device(qd, compact=False)]
        qa, qb = d.gen_queries(query)
        runs.append((qa.cuda(), qb.cuda()))
        where = {int(w): i for i, w in enumerate(kw)}
        want = np.array([values[where[int(w)]] if int(w) in where else np.zeros(e, np.int32) for w in query])
        want_found = np.array([int(w) in where for w in query])
        for qa, qb in runs:
            vals, found = d.reconstruct(d.eval_queries_device(qa), d.eval_queries_device(qb), qd)
            assert np.array_equal(found.cpu().numpy(), want_found)
            assert np.array_equal(vals.cpu().numpy(), want)
    finally:
        d.close()


@pytest.mark.parametrize("nq", [1, 5, 1000, 70000])
def test_device_plan_equals_host_locate(torch_cuda, nq):
    torch = torch_cuda
    n = 5000
    kw = keywords_of("random", n, 8)
    ctx = B.KeywordContext(kw, np.zeros((n, 1), np.int32), K.default_m(n), 0xFEED)
    try:
        rng = np.random.RandomState(nq)
        q = rng.randint(-(1 << 63), 1 << 63, nq, dtype=np.int64).astype(np.uint64)
        q[:min(nq, 3)] = np.array([0, M64 - 1, 1 << 63], np.uint64)[:min(nq, 3)]
        want = B.kwpir_locate(K.default_m(n), 0xFEED, q)
        assert np.array_equal(want, K.rows3(q, K.default_m(n), 0xFEED))
        qd = torch.as_tensor(q.view(np.int64)).cuda()
        out = torch.full((nq, 3), -7, dtype=torch.int64, device="cuda")
        ctx.plan_device(qd.data_ptr(), nq, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert np.array_equal(out.cpu().numpy(), want)
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_updates(torch_cuda, kind):
    torch = torch_cuda
    import dpf
    kw_args, suffix = KINDS[kind]
    n, E = 5003, 14
    prf = B.PRF_CHACHA20
    kw = keywords_of("random", n, 21)
    values = random_table(n, E, seed=9)
    d = dpf.KeywordDPF(prf, 0, seed=4242, **kw_args)
    d.eval_init(kw, values)
    try:
        rng = np.random.RandomState(3)
        query = kw[rng.choice(n, 64, replace=False)]
        qd = torch.as_tensor(query.view(np.int64)).cuda()
        qa, qb = d.gen_queries_device(qd)
        torch.cuda.synchronize()
        # a query batch in flight on another stream, enqueued before the update: it must see old values only
        s1 = torch.cuda.Stream()
        with torch.cuda.stream(s1):
            for _ in range(3):
                out_a = d.eval_queries_device(qa)
            out_b = d.eval_queries_device(qb)
        # every queried keyword and some repeats, the last occurrence winning
        upd = np.concatenate([query, query[:10], kw[:50]])
        new = random_table(len(upd), E, seed=77)
        d.update(upd, new)
        s1.synchronize()
        vals, found = d.reconstruct(out_a, out_b, qd)
        where = {int(w): i for i, w in enumerate(kw)}
        assert found.all()
        assert np.array_equal(vals.cpu().numpy(), values[[where[int(w)] for w in query]])
        expect = {int(w): values[where[int(w)]] for w in kw}
        for j, w in enumerate(upd):
            expect[int(w)] = new[j]
        check = np.concatenate([query, kw[:50], kw[rng.choice(n, 100, replace=False)]])
        cd = torch.as_tensor(check.view(np.int64)).cuda()
        ca, cb = d.gen_queries_device(cd)
        vals, found = d.reconstruct(d.eval_queries_device(ca), d.eval_queries_device(cb), cd)
        assert found.all()
        assert np.array_equal(vals.cpu().numpy(), np.array([expect[int(w)] for w in check]))
        # an absent keyword refuses the whole update; a grouped row update is refused
        before = dpf.dpf_cpp.kwpir_tags(d.buffers).numpy()
        with pytest.raises(RuntimeError, match="keyword 1 is not in the table"):
            d.update(np.array([kw[0], 1], np.uint64), np.full((2, E), 5, np.int32))
        with pytest.raises(RuntimeError, match="reserved"):
            d.update(np.array([M64], np.uint64), np.zeros((1, E), np.int32))
        vals, found = d.reconstruct(d.eval_queries_device(ca), d.eval_queries_device(cb), cd)
        assert np.array_equal(vals.cpu().numpy(), np.array([expect[int(w)] for w in check]))
        assert np.array_equal(dpf.dpf_cpp.kwpir_tags(d.buffers).numpy(), before)
        assert dpf.dpf_cpp.kwpir_build_stats(d.buffers)[0] >= 1
    finally:
        d.close()
    ctx = B.KeywordContext(kw[:100], values[:100], K.default_m(100), 1, **kw_args)
    try:
        L = B.lib()
        assert L.b200dpf_group_update_rows(ctx.handle, np.zeros(1, np.int32), np.zeros(1, np.int64), np.zeros(E + 2, np.int32), 1) == ESTATE
        assert "keyword-PIR context" in L.b200dpf_last_error().decode()
    finally:
        ctx.close()


@pytest.mark.parametrize("dev", [False, True])
def test_duplicate_and_reserved_keywords_are_refused(torch_cuda, dev):
    n = 1000
    kw = keywords_of("random", n, 5)
    values = np.zeros((n, 2), np.int32)
    for bad, msg in ((kw[17], "duplicate keywords"), (np.uint64(M64), "reserved")):
        k2 = kw.copy()
        k2[900] = bad
        with pytest.raises(B.B200DPFError, match=r"failed \(-1\).*" + msg):
            create(k2, values, K.default_m(n), 1, device_inputs=dev, torch=torch_cuda)
