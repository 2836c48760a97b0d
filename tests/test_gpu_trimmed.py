"""Trimmed tables (include/b200dpf.h "Trimmed tables") on the GPU: plain and grouped contexts of any row count,
for every kind of key, against an oracle built from the host share vectors:

    out[b][e] = sum over r < n of share_b[trimmed_alpha(r)] * table[r][e]   mod 2^32   (XOR-shared: XOR)

Every key's result is compared bit for bit (both servers' keys), and the pairs must reconstruct the selected rows."""
import ctypes as C
import functools
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
import plan_matrix  # noqa: E402
import sparse_oracle  # noqa: E402
import xor_oracle  # noqa: E402

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
KINDS = ("standard", "et", "xor")
SUFFIX = {"standard": "", "et": "_et", "xor": "_xor"}
LANE_BITS = {"standard": 0, "et": 2, "xor": 7}
EINVAL, ESTATE = -1, -4


def ctx_kw(kind):
    return dict(early_termination=kind == "et", xor=kind == "xor", trimmed=True)


def table_of(n, e, seed):
    return np.random.RandomState(seed).randint(-2 ** 31, 2 ** 31, size=(n, e), dtype=np.int64).astype(np.int32)


def rows_for(n, count, seed):
    """`count` rows of [0, n): both ends first, then random ones"""
    r = np.random.RandomState(seed).randint(0, n, size=count)
    r[:min(count, 2)] = [0, n - 1][:min(count, 2)]
    return r.astype(np.int64)


def keys_for(kind, n, rows, prf, seed=0):
    """both servers' keys for `rows` of a trimmed n-row table"""
    s = SUFFIX[kind]
    alphas = np.array([B.trimmed_alpha(int(r), n, s) for r in rows], np.int64)
    return plan_matrix.gen_keys(kind, B.trimmed_domain(n, s), alphas, prf, seed)


@functools.lru_cache(maxsize=None)
def key_index(n, kind):
    """trimmed_alpha(r) for every row r < n"""
    return np.array([B.trimmed_alpha(r, n, SUFFIX[kind]) for r in range(n)], np.int64)


def expected(kind, prf, keys, table):
    """the oracle above, from the host share vectors over the key domain"""
    order = key_index(table.shape[0], kind)
    keys = np.asarray(keys, np.int32).reshape(-1, 524)
    if kind == "xor":
        bits = np.stack([xor_oracle.unpack_bits(B.eval_cpu_xor(k, prf)) for k in keys])
        return xor_oracle.xor_rows(bits[:, order], table)
    ev = B.eval_cpu if kind == "standard" else B.eval_cpu_et
    shares = np.stack([ev(k, prf) for k in keys])
    return et_oracle.dot_u32(shares[:, order], table)


def check_pair(kind, prf, ka, kb, table, rows, ra, rb):
    assert np.array_equal(ra, expected(kind, prf, ka, table))
    assert np.array_equal(rb, expected(kind, prf, kb, table))
    assert np.array_equal(plan_matrix.reconstruct(kind, ra, rb), table[rows])


# ---- shapes: every kind and PRF, row counts from 1 to past 2^20, entry sizes, batch sizes ------------------

# (n, entry_size, batch)
SHAPES = [(1, 1, 1), (3, 5, 3), (255, 16, 31), (1000, 17, 32), (3001, 40, 33), (5000, 128, 17), (4096, 16, 512),
          (70001, 16, 512), ((1 << 20) + 1, 16, 3), (3 << 19, 1, 5), (1 << 16, 16, 64)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "n%d_e%d_b%d" % s)
def test_shapes(kind, prf, shape):
    n, e, batch = shape
    table = table_of(n, e, n + e)
    rows = rows_for(n, batch, batch)
    ka, kb = keys_for(kind, n, rows, prf, seed=n)
    ctx = B.Context(table, **ctx_kw(kind))
    try:
        assert ctx.trimmed and ctx.table_rows >= n
        check_pair(kind, prf, ka, kb, table, rows, ctx.eval(ka, prf), ctx.eval(kb, prf))
    finally:
        ctx.close()


# ---- the padding bound -----------------------------------------------------------------------------------

def bound_rows(n, kind):
    """the documented bound: n rounded up to 2^g, g = min(log2 N, max(log2 N - 7, b + m))"""
    N = B.trimmed_domain(n, SUFFIX[kind])
    logn = N.bit_length() - 1
    g = min(logn, max(logn - 7, LANE_BITS[kind] + (1 if kind == "xor" else 6)))
    return (n + (1 << g) - 1) >> g << g


@pytest.mark.parametrize("kind", KINDS)
def test_table_rows_within_bound(kind):
    for n in (1, 2, 63, 65, 700, 3000, 4097, 70001, (1 << 20) + 1, 3 << 19, (1 << 21) - (1 << 14)):
        ctx = B.Context(np.zeros((n, 1), np.int32), **ctx_kw(kind))
        try:
            assert ctx.table_rows == bound_rows(n, kind), n
            if n > (1 << (LANE_BITS[kind] + (1 if kind == "xor" else 6) + 7)):
                assert ctx.table_rows - n < n / 64, n
        finally:
            ctx.close()


# ---- options: the pairwise covering array of the tuning options, including forced s, top_log2, lane split --

@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("batch", [3, 40])
def test_options(kind, batch):
    n, e, prf = {"standard": 5000, "et": 9001, "xor": 70001}[kind], 40, B.PRF_AES128
    table = table_of(n, e, 7)
    rows = rows_for(n, batch, 8)
    ka, kb = keys_for(kind, n, rows, prf, seed=9)
    want_a, want_b = expected(kind, prf, ka, table), expected(kind, prf, kb, table)
    ctx = B.Context(table, **ctx_kw(kind))
    try:
        for row in plan_matrix.pairwise_rows():
            for name, value in row.items():
                ctx.set_option(name, value)
            assert np.array_equal(ctx.eval(ka, prf), want_a), row
            assert np.array_equal(ctx.eval(kb, prf), want_b), row
    finally:
        ctx.close()


# ---- every plain-context path ------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_paths(kind):
    n, e, batch, prf = 3001, 20, 40, B.PRF_CHACHA20
    table = table_of(n, e, 11)
    rows = rows_for(n, batch, 12)
    ka, kb = keys_for(kind, n, rows, prf, seed=13)
    want = expected(kind, prf, ka, table)
    ctx = B.Context(table, **ctx_kw(kind))
    try:
        assert np.array_equal(ctx.eval(ka, prf), want)
        assert np.array_equal(ctx.eval_gather(list(ka), prf), want)
        packed = b"".join(getattr(B, "key_pack" + SUFFIX[kind])(k) for k in ka)
        assert np.array_equal(ctx.eval_packed(packed, batch, prf), want)
        keys_dev = torch.from_numpy(ka).cuda()
        out = torch.zeros((batch, e), dtype=torch.int32, device="cuda")
        ctx.eval_device(keys_dev.data_ptr(), batch, prf, out.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), want)
        acc = torch.zeros_like(out)
        for _ in range(2):
            ctx.eval_device(keys_dev.data_ptr(), batch, prf, acc.data_ptr(), accumulate=True)
        torch.cuda.synchronize()
        twice = np.zeros_like(want) if kind == "xor" else (want.view(np.uint32) * np.uint32(2)).view(np.int32)
        assert np.array_equal(acc.cpu().numpy(), twice)
    finally:
        ctx.close()
    # the dpf_cpp binding: packed keys are sized by the key domain, not by the live rows
    import dpf
    d = dpf.DPF(prf=prf, trim=True, early_termination=kind == "et", xor=kind == "xor")
    try:
        d.eval_init(torch.from_numpy(table))
        assert np.array_equal(d.eval_gpu_compact(d.pack_keys(torch.from_numpy(ka))).numpy(), want)
    finally:
        d.close()


# ---- row updates by row number -----------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_update_rows(kind):
    n, e, batch, prf = 1001, 16, 33, B.PRF_AES128
    table = table_of(n, e, 21)
    ctx = B.Context(table, **ctx_kw(kind))
    try:
        rows = rows_for(n, batch, 22)
        ka, kb = keys_for(kind, n, rows, prf, seed=23)
        # host path, with a duplicate (the last one wins)
        idx = np.array([0, n - 1, 500, 500, 17], np.int64)
        new = table_of(len(idx), e, 24)
        ctx.update_rows(idx, new)
        for j, i in enumerate(idx):
            table[i] = new[j]
        check_pair(kind, prf, ka, kb, table, rows, ctx.eval(ka, prf), ctx.eval(kb, prf))
        # a row past n is refused and nothing is applied
        with pytest.raises(B.B200DPFError):
            ctx.update_rows(np.array([3, n], np.int64), table_of(2, e, 25))
        assert np.array_equal(ctx.eval(ka, prf), expected(kind, prf, ka, table))
        # device path on another stream: rows outside [0, n) are skipped; an evaluation enqueued before the update
        # sees the old rows, one after it the new rows
        idx2 = np.array([1, n, -1, 999, 1, n + 1000], np.int64)
        new2 = table_of(len(idx2), e, 26)
        old = table.copy()
        for j, i in enumerate(idx2):
            if 0 <= i < n:
                table[i] = new2[j]
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        keys_dev = torch.from_numpy(ka).cuda()
        before = torch.zeros((batch, e), dtype=torch.int32, device="cuda")
        after = torch.zeros_like(before)
        i_dev, r_dev = torch.from_numpy(idx2).cuda(), torch.from_numpy(new2).cuda()
        torch.cuda.synchronize()
        ctx.eval_device(keys_dev.data_ptr(), batch, prf, before.data_ptr(), stream=s1.cuda_stream)
        ctx.update_rows_device(i_dev.data_ptr(), r_dev.data_ptr(), len(idx2), stream=s2.cuda_stream)
        ctx.eval_device(keys_dev.data_ptr(), batch, prf, after.data_ptr(), stream=s1.cuda_stream)
        torch.cuda.synchronize()
        assert np.array_equal(before.cpu().numpy(), expected(kind, prf, ka, old))
        assert np.array_equal(after.cpu().numpy(), expected(kind, prf, ka, table))
        assert ctx.table_rows == bound_rows(n, kind)
    finally:
        ctx.close()


# ---- at a power of two, a trimmed context is a plain one whose table is permuted by trimmed_alpha ----------

@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("prf", [B.PRF_AES128, B.PRF_SALSA20])
def test_pow2_matches_permuted_plain_context(kind, prf):
    n, e, batch = 1 << 14, 16, 64
    table = table_of(n, e, 31)
    perm = np.empty_like(table)
    for r in range(n):
        perm[B.trimmed_alpha(r, n, SUFFIX[kind])] = table[r]
    rows = rows_for(n, batch, 32)
    ka, _ = keys_for(kind, n, rows, prf, seed=33)
    trimmed = B.Context(table, **ctx_kw(kind))
    plain = B.Context(perm, early_termination=kind == "et", xor=kind == "xor")
    try:
        assert trimmed.table_rows == n
        assert np.array_equal(trimmed.eval(ka, prf), plain.eval(ka, prf))
    finally:
        trimmed.close()
        plain.close()


# ---- bounds and refusals -----------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_refusals(kind):
    n, e, prf = 3000, 16, B.PRF_AES128
    ctx = B.Context(table_of(n, e, 41), **ctx_kw(kind))
    L = B.lib()
    try:
        N = B.trimmed_domain(n, SUFFIX[kind])
        wrong, _ = plan_matrix.gen_keys(kind, 2 * N, np.array([5], np.int64), prf)
        assert L.b200dpf_eval(ctx.handle, wrong, 1, prf, np.zeros((1, e), np.int32)) == EINVAL
        other = "et" if kind != "et" else "standard"
        foreign, _ = plan_matrix.gen_keys(other, B.trimmed_domain(n, SUFFIX[other]), np.array([5], np.int64), prf)
        assert L.b200dpf_eval(ctx.handle, foreign, 1, prf, np.zeros((1, e), np.int32)) == EINVAL
        ka, _ = keys_for(kind, n, [5], prf)
        keys_dev = torch.from_numpy(ka).cuda()
        out = torch.zeros((1, N), dtype=torch.int32, device="cuda")
        assert L.b200dpf_expand_device(ctx.handle, C.c_void_p(keys_dev.data_ptr()), 1, prf, C.c_void_p(out.data_ptr()),
                                       None) == ESTATE
        assert L.b200dpf_ctx_n(ctx.handle) == n
        assert L.b200dpf_ctx_trimmed(ctx.handle) == 1
    finally:
        ctx.close()
    plain = B.Context(table_of(256, 4, 42))
    try:
        assert L.b200dpf_ctx_trimmed(plain.handle) == 0 and plain.table_rows == 256
    finally:
        plain.close()


# ---- grouped contexts --------------------------------------------------------------------------------------

BINS = {"standard": [1, 3, 700, 1024, 3000, 64, 5000, 2],
        "et": [1, 9, 700, 1024, 3001, 8, 5000],
        "xor": [1, 300, 700, 1024, 3000, 256, 9000]}


def group_keys(kind, sizes, nq, prf, seed):
    """nq queries of one key per bin: int32 [nq, nbins, 524] for both servers, and the rows they select"""
    rng = np.random.RandomState(seed)
    rows = np.stack([rng.randint(0, n, size=nq) for n in sizes], axis=1).astype(np.int64)
    ka = np.zeros((nq, len(sizes), 524), np.int32)
    kb = np.zeros_like(ka)
    for g, n in enumerate(sizes):
        a, b = keys_for(kind, n, rows[:, g], prf, seed=seed + g)
        ka[:, g], kb[:, g] = a, b
    return ka, kb, rows


def group_expected(kind, prf, keys, tables):
    nq, nbins = keys.shape[:2]
    out = np.zeros((nq, nbins, tables[0].shape[1]), np.int32)
    for g in range(nbins):
        out[:, g] = expected(kind, prf, keys[:, g], tables[g])
    return out


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("prf", PRFS)
def test_grouped_paths(kind, prf):
    sizes, e, nq = BINS[kind], 20, 5
    tables = [table_of(n, e, 50 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **ctx_kw(kind))
    try:
        assert ctx.trimmed and ctx.table_rows == sum(bound_rows(n, kind) for n in sizes)
        ka, kb, rows = group_keys(kind, sizes, nq, prf, seed=prf)
        want_a, want_b = group_expected(kind, prf, ka, tables), group_expected(kind, prf, kb, tables)
        rec = plan_matrix.reconstruct(kind, want_a, want_b)
        for g in range(len(sizes)):
            assert np.array_equal(rec[:, g], tables[g][rows[:, g]])
        bins = np.tile(np.arange(len(sizes), dtype=np.int32), nq)
        # host path (keys in the caller's order, one bin each)
        flat = ka.reshape(-1, 524)
        assert np.array_equal(ctx.eval(flat, bins, prf).reshape(want_a.shape), want_a)
        assert np.array_equal(ctx.eval(kb.reshape(-1, 524), bins, prf).reshape(want_b.shape), want_b)
        # device keys, a shuffled key list
        perm = np.random.RandomState(3).permutation(len(bins))
        out = torch.zeros((len(bins), e), dtype=torch.int32, device="cuda")
        keys_dev = torch.from_numpy(np.ascontiguousarray(flat[perm])).cuda()
        ctx.eval_device(keys_dev.data_ptr(), bins[perm], prf, out.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), want_a.reshape(-1, e)[perm])
        # query batches, wire and compact
        qout = torch.zeros((nq, len(sizes), e), dtype=torch.int32, device="cuda")
        wire = torch.from_numpy(ka).cuda()
        ctx.eval_queries_device(wire.data_ptr(), nq, prf, qout.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(qout.cpu().numpy(), want_a)
        compact = torch.from_numpy(ctx.pack_queries(kb)).cuda()
        assert compact.shape[1] == ctx.query_bytes
        ctx.eval_queries_device(compact.data_ptr(), nq, prf, qout.data_ptr(), compact=True)
        torch.cuda.synchronize()
        assert np.array_equal(qout.cpu().numpy(), want_b)
        # row updates by row number
        upd_bins = np.array([0, 2, 2, len(sizes) - 1], np.int32)
        upd_idx = np.array([0, sizes[2] - 1, sizes[2] - 1, min(7, sizes[-1] - 1)], np.int64)
        new = table_of(len(upd_bins), e, 60)
        ctx.update_rows(upd_bins, upd_idx, new)
        for j in range(len(upd_bins)):
            tables[upd_bins[j]][upd_idx[j]] = new[j]
        assert np.array_equal(ctx.eval(flat, bins, prf).reshape(want_a.shape), group_expected(kind, prf, ka, tables))
        with pytest.raises(B.B200DPFError):
            ctx.update_rows(np.array([1], np.int32), np.array([sizes[1]], np.int64), new[:1])
        # a key for the bin's size rounded up by hand is the right one; a key for another domain is refused
        N1 = B.trimmed_domain(sizes[2], SUFFIX[kind])
        wrong, _ = plan_matrix.gen_keys(kind, 2 * N1, np.array([1], np.int64), prf)
        assert B.lib().b200dpf_group_eval(ctx.handle, wrong, np.array([2], np.int32), 1, prf,
                                          np.zeros((1, e), np.int32)) == EINVAL
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("prf", [B.PRF_AES128, B.PRF_CHACHA20])
def test_grouped_gen_queries_match_host_keygen(kind, prf):
    sizes, e, nq = BINS[kind], 8, 6
    tables = [table_of(n, e, 70 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **ctx_kw(kind))
    try:
        rng = np.random.RandomState(71)
        alphas = rng.randint(-2 ** 40, 2 ** 40, size=(nq, len(sizes))).astype(np.int64)
        alphas[0] = -1            # a true non-negative modulo: row n_g - 1
        seeds = rng.randint(0, 256, size=(nq, len(sizes), 44)).astype(np.uint8)
        a_dev, s_dev = torch.from_numpy(alphas).cuda(), torch.from_numpy(seeds).cuda()
        wa = torch.zeros((nq, len(sizes), 524), dtype=torch.int32, device="cuda")
        wb = torch.zeros_like(wa)
        ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, prf, wa.data_ptr(), wb.data_ptr())
        ca = torch.zeros((nq, ctx.query_bytes), dtype=torch.uint8, device="cuda")
        cb = torch.zeros_like(ca)
        ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, prf, ca.data_ptr(), cb.data_ptr(), compact=True)
        torch.cuda.synchronize()
        wa, wb, ca, cb = wa.cpu().numpy(), wb.cpu().numpy(), ca.cpu().numpy(), cb.cpu().numpy()
        s = SUFFIX[kind]
        gen = B.gen_batch_secure if kind == "standard" else getattr(B, "gen_batch" + s)
        rows = np.zeros((nq, len(sizes)), np.int64)
        for g, n in enumerate(sizes):
            rows[:, g] = alphas[:, g] % n
            idx = np.array([B.trimmed_alpha(int(r), n, s) for r in rows[:, g]], np.int64)
            ha, hb = gen(idx, B.trimmed_domain(n, s), seeds[:, g].tobytes(), prf)
            assert np.array_equal(wa[:, g], ha) and np.array_equal(wb[:, g], hb), g
        assert np.array_equal(ca, ctx.pack_queries(wa)) and np.array_equal(cb, ctx.pack_queries(wb))
        assert (rows[0] == np.array(sizes) - 1).all()
        # and they select those rows
        qa = torch.zeros((nq, len(sizes), e), dtype=torch.int32, device="cuda")
        qb = torch.zeros_like(qa)
        ctx.eval_queries_device(torch.from_numpy(ca).cuda().data_ptr(), nq, prf, qa.data_ptr(), compact=True)
        ctx.eval_queries_device(torch.from_numpy(cb).cuda().data_ptr(), nq, prf, qb.data_ptr(), compact=True)
        torch.cuda.synchronize()
        rec = plan_matrix.reconstruct(kind, qa.cpu().numpy(), qb.cpu().numpy())
        for g in range(len(sizes)):
            assert np.array_equal(rec[:, g], tables[g][rows[:, g]])
    finally:
        ctx.close()


# ---- one table past 2^29 rows ------------------------------------------------------------------------------

def test_large_table():
    """2^29 + 1 rows, E = 1: about 32 GiB of device table where padding to 2^30 rows would need 64.  The table is
    zero except on a support of rows; every key is checked from per-index walks of the C oracle over it."""
    import oracle as O
    n, prf, batch = (1 << 29) + 1, B.PRF_AES128, 32
    rng = np.random.RandomState(81)
    support = np.unique(np.concatenate([rng.randint(0, n, size=4000), [0, 1, n - 2, n - 1, 1 << 28, (1 << 28) - 1]]))
    vals = sparse_oracle.values(len(support), 1, 82)
    table = sparse_oracle.host_table(n, support, vals)
    rows = support[rng.randint(0, len(support), size=batch)]
    rows[:2] = [n - 1, 0]
    ka, kb = keys_for("standard", n, rows, prf, seed=83)
    ctx = B.Context(table, trimmed=True)
    del table
    try:
        assert ctx.table_rows == bound_rows(n, "standard") and ctx.table_rows < (1 << 29) * 1.02
        ra, rb = ctx.eval(ka, prf), ctx.eval(kb, prf)
    finally:
        ctx.close()
    orc = O.Oracle()
    idx = np.array([B.trimmed_alpha(int(r), n) for r in support], np.int64)
    for keys, got in ((ka, ra), (kb, rb)):
        assert np.array_equal(got, sparse_oracle.dot_u32(orc.eval_points(keys, prf, idx), vals))
    assert np.array_equal(sparse_oracle.sub_u32(ra, rb), vals[np.searchsorted(support, rows)])
