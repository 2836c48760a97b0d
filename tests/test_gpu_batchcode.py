"""Batch codes on the GPU (b200dpf_batchcode_*), for every kind of key with AES, ChaCha20 and Salsa20 across the
matrix: every bin row of small tables (and samples of large ones) reconstructs through b200dpf_group_eval to the table
row the layout puts there, from host and device tables; the device plan equals the host plan bit for bit; queries made
on the GPU in both formats, or on the host, and evaluated for both servers reconstruct the wanted rows; row updates
reach all three copies and leave a query enqueued before them on another stream alone; and the grouped row update is
refused."""
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
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
ESTATE = -4
KINDS = {"standard": ({}, ""), "et": ({"early_termination": True}, "_et"), "xor": ({"xor": True}, "_xor")}
PRFS = (B.PRF_AES128, B.PRF_CHACHA20, B.PRF_SALSA20)


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


def bin_rows(n, nbins):
    return [3 * ((n - j + nbins - 1) // nbins) for j in range(nbins)]


def host_gen(suffix, alphas, n, seeds, prf):
    return getattr(B, "gen_batch_secure" if suffix == "" else "gen_batch" + suffix)(alphas, n, seeds, prf)


def rec(suffix, a, b):
    a, b = a.astype(np.uint32), b.astype(np.uint32)
    return ((a ^ b) if suffix == "_xor" else (a - b)).astype(np.uint32).view(np.int32)


def bin_keys(suffix, sizes, bins, rows, prf, rng):
    """keys (both servers) for row rows[i] of bin bins[i]: the kind's key for trimmed_alpha(row, bin size)"""
    ka = np.zeros((len(bins), B.KEY_WORDS), np.int32)
    kb = np.zeros_like(ka)
    for size in sorted(set(sizes[b] for b in bins)):
        sel = [i for i, b in enumerate(bins) if sizes[b] == size]
        alphas = np.array([B.trimmed_alpha(int(rows[i]), size, suffix) for i in sel], np.int64)
        a, b = host_gen(suffix, alphas, B.trimmed_domain(size, suffix), rng.bytes(44 * len(sel)), prf)
        ka[sel], kb[sel] = a, b
    return ka, kb


def where_is(n, nbins, seed, rows):
    """{(bin, in-bin row): table row} for the copies of `rows`"""
    out = {}
    for r in rows:
        bs, rs = B.batchcode_locate(n, nbins, seed, int(r))
        for c in range(3):
            out[(int(bs[c]), int(rs[c]))] = int(r)
    return out


def make_ctx(torch, table, nbins, seed, kw, on_device):
    if not on_device:
        return B.BatchCodeContext(table, nbins, seed, **kw)
    t = torch.as_tensor(table).cuda()
    ctx = B.BatchCodeContext.__new__(B.BatchCodeContext)
    ctx.n, ctx.entry_size = table.shape
    ctx.kind = "_xor" if kw.get("xor") else "_et" if kw.get("early_termination") else ""
    ctx._trimmed = True
    ctx.handle = C.c_void_p()
    B._check(B.lib().b200dpf_batchcode_create(C.byref(ctx.handle), C.c_void_p(t.data_ptr()), ctx.n, ctx.entry_size, nbins, seed,
                                              0, B.KIND_IDS[ctx.kind]), "b200dpf_batchcode_create")
    return ctx


# (n, entry size, nbins, table in device memory, rows of the table checked: None = all)
LAYOUTS = [
    (300, 1, 1, False, None), (301, 16, 3, True, None), (4000, 40, 48, False, None), (3000, 128, 1536, True, None),
    ((1 << 20) + 1, 16, 48, False, 96), (3 << 18, 40, 1536, True, 96), (777, 16, 48, True, None),
]


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("case", range(len(LAYOUTS)))
def test_layout_every_bin_row(torch_cuda, kind, case):
    kw, suffix = KINDS[kind]
    n, E, nbins, on_device, sample = LAYOUTS[case]
    prf = PRFS[(case + list(KINDS).index(kind)) % len(PRFS)]
    rng = np.random.RandomState(case * 7 + len(kind))
    seed = int(rng.randint(0, 1 << 62))
    table = random_table(n, E, seed=case + 11)
    ctx = make_ctx(torch_cuda, table, nbins, seed, kw, on_device)
    try:
        assert ctx.layout == (n, nbins, seed)
        assert ctx.nbins == nbins
        sizes = bin_rows(n, nbins)
        rows = np.arange(n) if sample is None else np.unique(np.concatenate([rng.randint(0, n, sample), [0, n - 1]]))
        loc = where_is(n, nbins, seed, rows)
        if sample is None:
            assert len(loc) == 3 * n == sum(sizes)
        items = sorted(loc.items())
        bins = [b for (b, _), _ in items]
        brow = [r for (_, r), _ in items]
        ka, kb = bin_keys(suffix, sizes, bins, brow, prf, rng)
        bins = np.array(bins, np.int32)
        for j in range(0, len(bins), 4096):
            got = rec(suffix, ctx.eval(ka[j:j + 4096], bins[j:j + 4096], prf), ctx.eval(kb[j:j + 4096], bins[j:j + 4096], prf))
            want = table[[t for _, t in items[j:j + 4096]]]
            assert np.array_equal(got, want), "bin rows %d.. do not hold their table rows" % j
    finally:
        ctx.close()


@pytest.mark.parametrize("n,nbins,k,nq", [(1000, 1, 1, 5), (5000, 12, 8, 64), ((1 << 20) + 1, 48, 32, 200), (1 << 16, 192, 128, 40),
                                          (3000, 40, 100, 7), (1 << 20, 300, 200, 300)])
def test_device_plan_equals_host_plan(torch_cuda, n, nbins, k, nq):
    torch = torch_cuda
    rng = np.random.RandomState(n % 1000 + k)
    seed = int(rng.randint(0, 1 << 62))
    table = np.zeros((n, 1), np.int32)
    ctx = B.BatchCodeContext(table, nbins, seed)
    try:
        wanted = rng.randint(0, n, size=(nq, k)).astype(np.int64)
        wanted[::2, k // 2:] = wanted[::2, :k - k // 2]
        alphas, slots = B.batchcode_plan(n, nbins, seed, wanted)
        w = torch.as_tensor(wanted).cuda()
        a = torch.full((nq, nbins), 7, dtype=torch.int64, device="cuda")
        s = torch.full((nq, k), 7, dtype=torch.int32, device="cuda")
        ctx.plan_device(w.data_ptr(), nq, k, a.data_ptr(), s.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert np.array_equal(a.cpu().numpy(), alphas)
        assert np.array_equal(s.cpu().numpy(), slots)
        # rows outside [0, n) get slot -1 and leave the other rows' plan as it would be without them
        bad = wanted[:1].copy()
        bad[0, ::3] = np.where(np.arange(len(bad[0, ::3])) % 2 == 0, -1, n)
        keep = (bad[0] >= 0) & (bad[0] < n)
        w = torch.as_tensor(bad).cuda()
        ctx.plan_device(w.data_ptr(), 1, k, a.data_ptr(), s.data_ptr(), 0)
        got_s = s[0].cpu().numpy()
        assert (got_s[~keep] == -1).all()
        if keep.any():
            ra, rs = B.batchcode_plan(n, nbins, seed, bad[:, keep])
            assert np.array_equal(got_s[keep], rs[0])
            assert np.array_equal(a[0].cpu().numpy(), ra[0])
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("prf", PRFS)
def test_queries_reconstruct_wanted_rows(torch_cuda, kind, prf):
    torch = torch_cuda
    import dpf
    kw, suffix = KINDS[kind]
    n, E, k, nq = 20011, 24, 32, 9
    nbins = 48
    table = random_table(n, E, seed=5)
    d = dpf.BatchCodeDPF(prf, 0, nbins, seed=12345 + prf, **kw)
    d.eval_init(torch.as_tensor(table))
    try:
        rng = np.random.RandomState(prf)
        wanted = rng.randint(0, n, size=(nq, k)).astype(np.int64)
        wanted[0, 1] = wanted[0, 0]
        runs = []
        wd = torch.as_tensor(wanted).cuda()
        for compact in (True, False):
            qa, qb, slots = d.gen_queries_device(wd, compact=compact)
            runs.append((qa, qb, slots))
        qa, qb, slots = d.gen_queries(torch.as_tensor(wanted))
        runs.append((qa.cuda(), qb.cuda(), slots))
        host_slots = d.plan(wanted)[1]
        for qa, qb, slots in runs:
            assert np.array_equal(torch.as_tensor(slots).cpu().numpy(), host_slots.numpy())
            rows, found = d.reconstruct(d.eval_queries_device(qa), d.eval_queries_device(qb), slots)
            rows, found = rows.cpu().numpy(), found.cpu().numpy()
            assert found.mean() > 0.9
            assert np.array_equal(rows[found], table[wanted[found]])
            assert not rows[~found].any()
    finally:
        d.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_update_rows_every_copy_and_ordering(torch_cuda, kind):
    torch = torch_cuda
    kw, suffix = KINDS[kind]
    n, E, nbins = 5003, 16, 24
    prf = B.PRF_CHACHA20
    seed = 4242
    table = random_table(n, E, seed=9)
    ctx = B.BatchCodeContext(table, nbins, seed, **kw)
    try:
        rng = np.random.RandomState(3)
        sizes = bin_rows(n, nbins)
        # a query batch in flight on another stream, enqueued before the update: it must see old rows only
        wanted = rng.randint(0, n, size=(64, 16)).astype(np.int64)
        alphas, slots = B.batchcode_plan(n, nbins, seed, wanted)
        ka, kb = np.zeros((64, nbins, B.KEY_WORDS), np.int32), np.zeros((64, nbins, B.KEY_WORDS), np.int32)
        for g in range(nbins):
            ka[:, g], kb[:, g] = bin_keys(suffix, sizes, [g] * 64, alphas[:, g], prf, rng)
        s1 = torch.cuda.Stream()
        keys_a, keys_b = torch.as_tensor(ka).cuda(), torch.as_tensor(kb).cuda()
        torch.cuda.synchronize()
        out_a = torch.empty((64, nbins, E), dtype=torch.int32, device="cuda")
        out_b = torch.empty_like(out_a)
        with torch.cuda.stream(s1):
            for _ in range(3):
                ctx.eval_queries_device(keys_a.data_ptr(), 64, prf, out_a.data_ptr(), s1.cuda_stream)
            ctx.eval_queries_device(keys_b.data_ptr(), 64, prf, out_b.data_ptr(), s1.cuda_stream)
        # the update: every wanted row and some repeats, the last occurrence winning
        idx = np.concatenate([wanted.reshape(-1)[:200], wanted.reshape(-1)[:50]])
        new = rng.randint(-2 ** 31, 2 ** 31, size=(len(idx), E), dtype=np.int64).astype(np.int32)
        ctx.update_rows(idx, new)
        s1.synchronize()
        a, b = out_a.cpu().numpy(), out_b.cpu().numpy()
        for q in range(64):
            for i in range(16):
                if slots[q, i] >= 0:
                    assert np.array_equal(rec(suffix, a[q, slots[q, i]], b[q, slots[q, i]]), table[wanted[q, i]])
        expect = {}
        for j, r in enumerate(idx):
            expect[int(r)] = new[j]
        loc = where_is(n, nbins, seed, sorted(expect))
        items = sorted(loc.items())
        bins = np.array([b for (b, _), _ in items], np.int32)
        qa, qb = bin_keys(suffix, sizes, list(bins), [r for (_, r), _ in items], prf, rng)
        got = rec(suffix, ctx.eval(qa, bins, prf), ctx.eval(qb, bins, prf))
        assert np.array_equal(got, np.array([expect[t] for _, t in items]))
        # rows not updated are unchanged in every copy
        other = [r for r in range(0, n, 97) if r not in expect]
        loc = where_is(n, nbins, seed, other)
        items = sorted(loc.items())
        bins = np.array([b for (b, _), _ in items], np.int32)
        qa, qb = bin_keys(suffix, sizes, list(bins), [r for (_, r), _ in items], prf, rng)
        assert np.array_equal(rec(suffix, ctx.eval(qa, bins, prf), ctx.eval(qb, bins, prf)), table[[t for _, t in items]])
        # a grouped update of one copy is refused, and an index out of range applies nothing
        L = B.lib()
        assert L.b200dpf_group_update_rows(ctx.handle, np.zeros(1, np.int32), np.zeros(1, np.int64), np.zeros(E, np.int32), 1) == ESTATE
        assert "batch-code context" in L.b200dpf_last_error().decode()
        with pytest.raises(B.B200DPFError, match="out of range"):
            ctx.update_rows([0, n], np.zeros((2, E), np.int32))
    finally:
        ctx.close()
