"""Every server's whole answer, not only the pair's reconstruction, on the query and update paths of trimmed grouped
contexts: batch codes, keyword PIR, queries generated on the GPU and device-resident bin lists.

Away from the selected row both servers hold equal seeds, so a row dropped, counted twice, read from a neighbour, or an
update that also lands in another slot or copy, changes both answers alike and cancels in a - b.  Here each server's
[Q, nbins, E] answer must equal tests/server_ref.py's exact reference bit for bit, over the bins restated from the
header (tests/batchcode_ref.py, tests/kwpir_ref.py): with a random key every live row of a bin carries a pseudo-random
weight, so one comparison covers the whole bin.  The references come from the keys the GPU was given (wire keys
downloaded, compact ones unpacked), so the evaluation is checked apart from the key generation.  Every pair must still
reconstruct its row.  The selected rows include the first and the last row of each bin and rows whose key paths turn
at every level."""
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
import batchcode_ref as BC  # noqa: E402
import kwpir_ref as K  # noqa: E402
import plan_matrix as PM  # noqa: E402
import server_ref as S  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1
KINDS = {"standard": {}, "et": {"early_termination": True}, "xor": {"xor": True}}
PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


def host(t):
    return t.cpu().numpy()


def wire_keys(kind, bin_rows, q, trimmed=True):
    """a query batch as host wire keys: int32 [Q, nbins, 524] from wire keys or compact queries (CUDA or host)"""
    q = q.cpu().numpy() if hasattr(q, "cpu") else np.asarray(q)
    if q.dtype == np.uint8:
        return S.unpack_queries(kind, bin_rows, q, trimmed)
    return q.astype(np.int32).reshape(q.shape[0], len(bin_rows), B.KEY_WORDS)


def edge_alphas(kind, bin_rows, trimmed=True):
    """int64 [4, nbins]: query 0 selects row 0 of every bin, query 1 the last row, queries 2 and 3 the rows whose key
    paths alternate (server_ref.edge_rows)"""
    return np.array([S.edge_rows(r, kind, trimmed) for r in bin_rows], np.int64).T.copy()


def check_answers(kind, prf, keys_a, keys_b, out_a, out_b, tables, trimmed=True, what=""):
    """each server's answers equal the reference; returns the references"""
    want_a = S.query_answers(kind, prf, keys_a, tables, trimmed)
    want_b = S.query_answers(kind, prf, keys_b, tables, trimmed)
    for server, got, want in (("A", out_a, want_a), ("B", out_b, want_b)):
        bad = np.argwhere((got != want).any(axis=-1))
        assert len(bad) == 0, "%s server %s: %d (query, bin) answers differ, first %s" % (what, server, len(bad), bad[:4].tolist())
    return want_a, want_b


# ---- batch codes ------------------------------------------------------------------------------------------------

# (n, E, nbins, queries, prf): bins of two sizes wherever nbins does not divide n
BATCHCODE = [
    (20011, 17, 48, 33, B.PRF_AES128),            # bins of 1251 and 1248 rows
    (3001, 16, 1536, 1, B.PRF_CHACHA20),          # bins of 6 and 3 rows
    ((1 << 15) + 5, 1, 1, 31, B.PRF_SALSA20),     # one bin of 98,319 rows
    (5003, 128, 48, 512, B.PRF_CHACHA20),         # bins of 315 and 312 rows
    (777, 40, 48, 33, B.PRF_DUMMY),               # bins of 51 and 48 rows
]


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("case", range(len(BATCHCODE)), ids=lambda c: "n%d_e%d_bins%d_q%d" % BATCHCODE[c][:4])
def test_batchcode_every_server_answer(torch, kind, case):
    """queries from the host client, the device client in both formats and the device generator at the edge rows,
    evaluated by eval_queries_device, by the host eval with explicit bins and by eval_gpu_device_bins"""
    import dpf
    n, E, nbins, nq, prf = BATCHCODE[case]
    rng = np.random.RandomState(case * 3 + len(kind))
    seed = int(rng.randint(0, 1 << 62))
    table = random_table(n, E, seed=case + 100)
    bins = BC.bins(table, n, nbins, seed)
    sizes = [b.shape[0] for b in bins]
    d = dpf.BatchCodeDPF(prf, 0, nbins, seed=seed, **KINDS[kind])
    d.eval_init(torch.as_tensor(table))
    try:
        assert d.bin_sizes == sizes
        k = max(1, 2 * nbins // 3)
        wanted = rng.randint(0, n, size=(nq, k)).astype(np.int64)
        wanted[0, :min(k, 2)] = [0, n - 1][:min(k, 2)]
        wd = torch.as_tensor(wanted).cuda()
        runs = []
        qa, qb, slots = d.gen_queries(torch.as_tensor(wanted))
        runs.append(("host client", qa.cuda(), qb.cuda(), slots))
        for compact in (True, False):
            qa, qb, slots = d.gen_queries_device(wd, compact=compact)
            runs.append(("device client, compact=%s" % compact, qa, qb, slots))
        alphas = edge_alphas(kind, sizes)
        qa, qb = dpf.BinnedDPF.gen_queries_device(d, torch.as_tensor(alphas).cuda(), compact=False)
        runs.append(("edge rows", qa, qb, None))
        for what, qa, qb, slots in runs:
            out_a, out_b = d.eval_queries_device(qa), d.eval_queries_device(qb)
            ka, kb = wire_keys(kind, sizes, qa), wire_keys(kind, sizes, qb)
            want_a, want_b = check_answers(kind, prf, ka, kb, host(out_a), host(out_b), bins, what=what)
            if slots is None:
                rec = PM.reconstruct(kind, want_a, want_b)
                for g in range(nbins):
                    assert np.array_equal(rec[:, g], bins[g][alphas[:, g]]), (what, g)
            else:
                rows, found = d.reconstruct(out_a, out_b, slots)
                rows, found = host(rows), host(found)
                assert found.mean() > 0.9
                assert np.array_equal(rows[found], table[wanted[found]]), what
            if what in ("host client", "edge rows"):
                # the same keys as one flat list: on the host path, and from device bin lists in a shuffled order
                flat_a, flat_b = ka.reshape(-1, B.KEY_WORDS), kb.reshape(-1, B.KEY_WORDS)
                ids = np.tile(np.arange(nbins, dtype=np.int32), ka.shape[0])
                assert np.array_equal(host(d.eval_gpu(torch.as_tensor(flat_a), ids)), want_a.reshape(-1, E)), what
                perm = rng.permutation(len(ids))
                ra = d.eval_gpu_device_bins(torch.as_tensor(flat_b[perm]).cuda(), torch.as_tensor(ids[perm]).cuda())
                assert np.array_equal(host(ra), want_b.reshape(-1, E)[perm]), what
    finally:
        d.close()


# ---- keyword PIR ------------------------------------------------------------------------------------------------

KEYWORD = [(kind, prf, e, (1.15, 1.3)[(i + j) % 2]) for kind in KINDS for i, prf in enumerate((B.PRF_AES128, B.PRF_CHACHA20))
           for j, e in enumerate((1, 14, 16, 125))]


def keywords_of(n, seed):
    """n distinct even keywords: odd ones are absent"""
    rng = np.random.RandomState(seed)
    kw = np.unique(rng.randint(0, 1 << 62, 2 * n + 8, dtype=np.int64).astype(np.uint64) * np.uint64(2))[:n]
    rng.shuffle(kw)
    return kw


@pytest.mark.parametrize("kind,prf,e,load", KEYWORD)
def test_keyword_every_server_answer(torch, kind, prf, e, load):
    """present and absent keywords through the host client, the device client in both formats and the device
    generator at the edge rows: each server's answer on all three bins equals the reference over kwpir_ref.bins, which
    also holds every empty slot at zero.  Value size 16 takes the 18-column path past one 16-column pass."""
    import dpf
    n = 3000
    kw = keywords_of(n, e)
    values = random_table(n, e, seed=e + 7)
    d = dpf.KeywordDPF(prf, 0, seed=99 + e, expansion=load, **KINDS[kind])
    d.eval_init(kw, values)
    try:
        m = d.m
        assert m == K.default_m(n, load)
        bins = K.bins(kw, values, m, d.seed)
        rng = np.random.RandomState(e)
        present = kw[rng.choice(n, 24, replace=False)]
        absent = np.array([1, 3, (1 << 63) + 1, M64 - 2] + list(rng.randint(0, 1 << 62, 4).astype(np.uint64) * np.uint64(2) + np.uint64(1)),
                          np.uint64)
        query = np.concatenate([present[:12], absent, present[12:]])
        qd = torch.as_tensor(query.view(np.int64)).cuda()
        runs = [("host client",) + tuple(x.cuda() for x in d.gen_queries(query))]
        for compact in (True, False):
            runs.append(("device client, compact=%s" % compact,) + d.gen_queries_device(qd, compact=compact))
        alphas = edge_alphas(kind, [m] * 3)
        runs.append(("edge rows",) + dpf.BinnedDPF.gen_queries_device(d, torch.as_tensor(alphas).cuda(), compact=True))
        where = {int(w): i for i, w in enumerate(kw)}
        want_vals = np.array([values[where[int(w)]] if int(w) in where else np.zeros(e, np.int32) for w in query])
        for what, qa, qb in runs:
            out_a, out_b = d.eval_queries_device(qa), d.eval_queries_device(qb)
            ka, kb = wire_keys(kind, [m] * 3, qa), wire_keys(kind, [m] * 3, qb)
            want_a, want_b = check_answers(kind, prf, ka, kb, host(out_a), host(out_b), bins, what=what)
            rec = PM.reconstruct(kind, want_a, want_b)
            if what == "edge rows":
                for c in range(3):
                    assert np.array_equal(rec[:, c], bins[c][alphas[:, c]])
                continue
            vals, found = d.reconstruct(out_a, out_b, qd)
            assert np.array_equal(host(found), np.array([int(w) in where for w in query])), what
            assert np.array_equal(host(vals), want_vals), what
    finally:
        d.close()


# ---- updates ----------------------------------------------------------------------------------------------------

def eval_pair(d, qa, qb):
    return host(d.eval_queries_device(qa)), host(d.eval_queries_device(qb))


@pytest.mark.parametrize("kind", list(KINDS))
def test_batchcode_updates_every_bin_row(torch, kind):
    """after update_rows (repeats included, the last occurrence winning), every row of every bin equals the restated
    layout of the updated table; a batch enqueued on another stream before the update answers from the old table; a
    refused update leaves every bin as it was"""
    import dpf
    n, E, nbins, prf = 5003, 16, 24, B.PRF_CHACHA20
    seed = 4242
    table = random_table(n, E, seed=9)
    d = dpf.BatchCodeDPF(prf, 0, nbins, seed=seed, **KINDS[kind])
    d.eval_init(torch.as_tensor(table))
    try:
        sizes = d.bin_sizes
        rng = np.random.RandomState(3)
        nq = 8                      # XOR-shared keys weigh a row 0 or 1: eight queries miss a changed row with p = 2^-8
        wanted = rng.randint(0, n, size=(nq, 16)).astype(np.int64)
        qa, qb, _ = d.gen_queries(torch.as_tensor(wanted))
        qa, qb = qa.cuda(), qb.cuda()
        ka, kb = host(qa), host(qb)
        old = BC.bins(table, n, nbins, seed)
        want_old = (S.query_answers(kind, prf, ka, old), S.query_answers(kind, prf, kb, old))
        torch.cuda.synchronize()
        s1 = torch.cuda.Stream()
        with torch.cuda.stream(s1):
            for _ in range(3):
                out_a = d.eval_queries_device(qa)
            out_b = d.eval_queries_device(qb)
        # the rows whose copies sit first or last in some bin, the wanted rows, and repeats
        ends = [r for r in range(n) if any(row in (0, sizes[b] - 1) for b, row in zip(*BC.locate(n, nbins, seed, r)))][:40]
        idx = np.concatenate([ends, wanted.reshape(-1)[:100], wanted.reshape(-1)[:30], [0, n - 1, 0]]).astype(np.int64)
        new = rng.randint(-2 ** 31, 2 ** 31, size=(len(idx), E), dtype=np.int64).astype(np.int32)
        d.update_rows(idx, new)
        s1.synchronize()
        for server, got, want in (("A", host(out_a), want_old[0]), ("B", host(out_b), want_old[1])):
            assert np.array_equal(got, want), "server %s: the batch enqueued before the update saw it" % server
        for j, r in enumerate(idx):
            table[r] = new[j]
        updated = BC.bins(table, n, nbins, seed)
        ca, cb, _ = d.gen_queries_device(torch.as_tensor(rng.randint(0, n, size=(nq, 16)).astype(np.int64)).cuda())
        cka, ckb = wire_keys(kind, sizes, ca), wire_keys(kind, sizes, cb)
        out = eval_pair(d, ca, cb)
        check_answers(kind, prf, cka, ckb, out[0], out[1], updated, what="after the update")
        ea, eb = dpf.BinnedDPF.gen_queries_device(d, torch.as_tensor(edge_alphas(kind, sizes)).cuda(), compact=False)
        out_e = eval_pair(d, ea, eb)
        check_answers(kind, prf, host(ea), host(eb), out_e[0], out_e[1], updated, what="edge rows after the update")
        # refused: an index out of range, or a negative one, applies nothing anywhere
        for bad in ([1, n], [-1, 2]):
            with pytest.raises(Exception, match="out of range"):
                d.update_rows(np.array(bad, np.int64), np.full((2, E), 7, np.int32))
            again = eval_pair(d, ca, cb)
            assert np.array_equal(again[0], out[0]) and np.array_equal(again[1], out[1]), bad
    finally:
        d.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_keyword_updates_every_bin_row(torch, kind):
    """after KeywordDPF.update (repeats included, the last occurrence winning), every slot of the three bins equals
    kwpir_ref.bins of the updated values, empty slots zero; a batch enqueued on another stream before the update
    answers from the old values; a refused update (an absent or reserved keyword) leaves every slot as it was"""
    import dpf
    n, E, prf = 5003, 14, B.PRF_CHACHA20
    kw = keywords_of(n, 21)
    values = random_table(n, E, seed=9)
    d = dpf.KeywordDPF(prf, 0, seed=4242, **KINDS[kind])
    d.eval_init(kw, values)
    try:
        m, seed = d.m, d.seed
        rng = np.random.RandomState(3)
        nq = 8
        query = kw[rng.choice(n, nq, replace=False)]
        qa, qb = d.gen_queries_device(torch.as_tensor(query.view(np.int64)).cuda(), compact=False)
        old = K.bins(kw, values, m, seed)
        want_old = (S.query_answers(kind, prf, host(qa), old), S.query_answers(kind, prf, host(qb), old))
        torch.cuda.synchronize()
        s1 = torch.cuda.Stream()
        with torch.cuda.stream(s1):
            for _ in range(3):
                out_a = d.eval_queries_device(qa)
            out_b = d.eval_queries_device(qb)
        # the items in the first and last slot of each bin, queried ones, and repeats
        _, owner = K.place(kw, m, seed)
        ends = [owner[c * m + r] for c in range(3) for r in (0, m - 1) if owner[c * m + r] >= 0]
        upd = np.concatenate([kw[ends], query, kw[:200], query[:4], kw[:20]])
        new = random_table(len(upd), E, seed=77)
        d.update(upd, new)
        s1.synchronize()
        for server, got, want in (("A", host(out_a), want_old[0]), ("B", host(out_b), want_old[1])):
            assert np.array_equal(got, want), "server %s: the batch enqueued before the update saw it" % server
        where = {int(w): i for i, w in enumerate(kw)}
        for j, w in enumerate(upd):
            values[where[int(w)]] = new[j]
        updated = K.bins(kw, values, m, seed)
        probe = kw[rng.choice(n, nq, replace=False)]
        ca, cb = d.gen_queries_device(torch.as_tensor(probe.view(np.int64)).cuda(), compact=True)
        cka, ckb = wire_keys(kind, [m] * 3, ca), wire_keys(kind, [m] * 3, cb)
        out = eval_pair(d, ca, cb)
        check_answers(kind, prf, cka, ckb, out[0], out[1], updated, what="after the update")
        ea, eb = dpf.BinnedDPF.gen_queries_device(d, torch.as_tensor(edge_alphas(kind, [m] * 3)).cuda(), compact=False)
        out_e = eval_pair(d, ea, eb)
        check_answers(kind, prf, host(ea), host(eb), out_e[0], out_e[1], updated, what="edge rows after the update")
        for bad, msg in ((np.array([kw[0], 1], np.uint64), "keyword 1 is not in the table"), (np.array([M64], np.uint64), "reserved")):
            with pytest.raises(RuntimeError, match=msg):
                d.update(bad, np.full((len(bad), E), 5, np.int32))
            again = eval_pair(d, ca, cb)
            assert np.array_equal(again[0], out[0]) and np.array_equal(again[1], out[1]), msg
        assert np.array_equal(dpf.dpf_cpp.kwpir_tags(d.buffers).numpy().view(np.uint64), K.tags(kw, owner, m))
    finally:
        d.close()


# ---- queries generated on the GPU, on plain grouped contexts -------------------------------------------------------

# per kind: bins of powers of two (of several depths) and trimmed bins
GROUPED = {
    "standard": ([2, 64, 1 << 10, 8, 1 << 14], [1, 3, 700, 1024, 3000, 64, 5000, 2]),
    "et": ([8, 64, 1 << 10, 32, 1 << 14], [1, 9, 700, 1024, 3001, 8, 5000]),
    "xor": ([256, 1 << 12, 512, 1 << 10, 1 << 14], [1, 300, 700, 1024, 3000, 256, 9000]),
}


def gen_and_eval(torch, ctx, alphas, prf, compact, st):
    """gen_queries_device then eval_queries_device of both servers on stream st with no sync in between: (host wire
    keys A, B, answers A, B)"""
    nq, nbins = alphas.shape
    size = nq * ctx.query_bytes if compact else nq * nbins * B.KEY_WORDS * 4
    with torch.cuda.stream(st):
        a_dev = torch.from_numpy(alphas).cuda()
        s_dev = torch.randint(0, 256, (nq, nbins, 44), dtype=torch.uint8, device="cuda")
        qa = torch.empty(size, dtype=torch.uint8, device="cuda")
        qb = torch.empty_like(qa)
        outs = [torch.full((nq, nbins, ctx.entry_size), -1, dtype=torch.int32, device="cuda") for _ in range(2)]
    ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, prf, qa.data_ptr(), qb.data_ptr(), st.cuda_stream, compact=compact)
    for q, o in zip((qa, qb), outs):
        ctx.eval_queries_device(q.data_ptr(), nq, prf, o.data_ptr(), st.cuda_stream, compact=compact)
    st.synchronize()
    kind = {"": "standard", "_et": "et", "_xor": "xor"}[ctx.kind]
    trimmed = ctx._trimmed
    if compact:
        keys = [S.unpack_queries(kind, ctx.bin_rows, host(q).reshape(nq, -1), trimmed) for q in (qa, qb)]
    else:
        keys = [host(q).view(np.int32).reshape(nq, nbins, B.KEY_WORDS) for q in (qa, qb)]
    return keys[0], keys[1], host(outs[0]), host(outs[1])


@pytest.mark.parametrize("trimmed", (False, True), ids=("pow2", "trimmed"))
@pytest.mark.parametrize("kind", list(KINDS))
def test_generated_queries_every_server_answer(torch, kind, trimmed):
    """every PRF, both formats: the keys the GPU generated, evaluated on the same stream, answer as the reference of
    those keys says, on every row of every bin"""
    sizes = GROUPED[kind][1 if trimmed else 0]
    e = 5
    tables = [random_table(n, e, seed=30 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, trimmed=trimmed, **KINDS[kind])
    st = torch.cuda.Stream()
    try:
        for i, prf in enumerate(PRFS):
            nq = (33, 4, 31, 1)[i]
            rng = np.random.RandomState(prf)
            alphas = np.stack([rng.randint(0, n, size=nq) for n in sizes], axis=1).astype(np.int64)
            edges = edge_alphas(kind, sizes, trimmed)
            alphas[:min(nq, 4)] = edges[:min(nq, 4)]
            ka, kb, ra, rb = gen_and_eval(torch, ctx, alphas, prf, compact=i % 2 == 0, st=st)
            want_a, want_b = check_answers(kind, prf, ka, kb, ra, rb, tables, trimmed, what="prf %d" % prf)
            rec = PM.reconstruct(kind, want_a, want_b)
            for g in range(len(sizes)):
                assert np.array_equal(rec[:, g], tables[g][alphas[:, g]]), (prf, g)
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_generated_queries_throughput_shape(torch, kind):
    """256 bins of 2^10 rows, AES, compact, generated twice on one stream and evaluated: every answer of both servers"""
    nbins, n, nq, e = 256, 1 << 10, 64, 4
    tables = [random_table(n, e, seed=50 + g) for g in range(nbins)]
    ctx = B.GroupContext(tables, **KINDS[kind])
    st = torch.cuda.Stream()
    try:
        rng = np.random.RandomState(7)
        for rnd in range(2):
            alphas = rng.randint(0, n, size=(nq, nbins)).astype(np.int64)
            alphas[:4] = edge_alphas(kind, [n] * nbins, False)
            ka, kb, ra, rb = gen_and_eval(torch, ctx, alphas, B.PRF_AES128, compact=True, st=st)
            check_answers(kind, B.PRF_AES128, ka, kb, ra, rb, tables, False, what="round %d" % rnd)
    finally:
        ctx.close()


# ---- device-resident bin lists ------------------------------------------------------------------------------------

def list_keys(kind, sizes, bins, prf, rng, trimmed=False):
    """both servers' keys for random rows of bins[j] (the first and last rows among them); keys whose bin is out of
    range are keys of bin 0"""
    home = np.where((bins >= 0) & (bins < len(sizes)), bins, 0)
    ka = np.zeros((len(bins), B.KEY_WORDS), np.int32)
    kb = np.zeros_like(ka)
    rows = np.array([rng.randint(0, sizes[g]) for g in home], np.int64)
    rows[:2 * len(sizes):2] = 0
    rows[1:2 * len(sizes):2] = np.array([sizes[g] - 1 for g in home[1:2 * len(sizes):2]])
    for n in sorted(set(sizes[g] for g in home)):
        sel = np.flatnonzero(np.array([sizes[g] for g in home]) == n)
        idx = S.key_index(n, kind, trimmed)[rows[sel]]
        ka[sel], kb[sel] = PM.gen_keys(kind, S.domain(n, kind, trimmed), idx, prf, seed=int(rng.randint(1 << 30)))
    return ka, kb, rows


def eval_bins(torch, ctx, keys, bins, prf):
    out = torch.full((len(keys), ctx.entry_size), -1, dtype=torch.int32, device="cuda")
    bad = torch.full((1,), 12345, dtype=torch.int64, device="cuda")
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys)).cuda()          # held until the call has run
    bins_dev = torch.from_numpy(np.ascontiguousarray(bins, np.int32)).cuda()
    st = torch.cuda.current_stream()
    ctx.eval_device_bins(keys_dev.data_ptr(), bins_dev.data_ptr(), len(keys), prf, out.data_ptr(), bad.data_ptr(), st.cuda_stream)
    st.synchronize()
    return host(out), int(bad.item())


def check_list(torch, kind, ctx, tables, bins, prf, rng, trimmed=False):
    sizes = [t.shape[0] for t in tables]
    ka, kb, rows = list_keys(kind, sizes, bins, prf, rng, trimmed)
    good = (bins >= 0) & (bins < len(tables))
    outs = []
    for server, keys in (("A", ka), ("B", kb)):
        got, bad = eval_bins(torch, ctx, keys, bins, prf)
        assert bad == int((~good).sum())
        want = S.grouped_answers(kind, prf, keys, bins, tables, trimmed)
        wrong = np.flatnonzero((got != want).any(axis=1))
        assert len(wrong) == 0, "server %s: %d keys differ, first at %s (bins %s)" % (server, len(wrong), wrong[:4].tolist(),
                                                                                     bins[wrong[:4]].tolist())
        outs.append(got)
    rec = PM.reconstruct(kind, outs[0][good], outs[1][good])
    assert np.array_equal(rec, np.stack([tables[g][r] for g, r in zip(bins[good], rows[good])]))


MIXES = ["uniform", "one_bin", "one_per_bin", "many_empty", "counts_31_32_33", "tiled"]


def make_bins(mix, nbins, rng):
    if mix == "uniform":
        return rng.randint(0, nbins, size=700).astype(np.int32)
    if mix == "one_bin":
        return np.full(1000, nbins // 2, np.int32)
    if mix == "one_per_bin":
        return rng.permutation(nbins).astype(np.int32)
    if mix == "many_empty":
        return rng.choice([1, nbins // 3, nbins - 1], size=300).astype(np.int32)
    if mix == "counts_31_32_33":
        b = np.repeat(np.arange(nbins, dtype=np.int32), [(31, 32, 33)[g % 3] for g in range(nbins)])
        return rng.permutation(b).astype(np.int32)
    return np.tile(np.arange(nbins, dtype=np.int32), 9)


@pytest.mark.parametrize("prf", [B.PRF_CHACHA20, B.PRF_AES128])
@pytest.mark.parametrize("kind", list(KINDS))
def test_device_bin_lists_every_server_answer(torch, kind, prf):
    """the bin mixes on bins of one size, mixed sizes with out-of-range bins (their keys answer zero and are counted),
    and trimmed bins: every key of both servers against the reference"""
    rng = np.random.RandomState(prf + 10 * len(kind))
    n = 1 << 10
    tables = [random_table(n, 16, seed=7 * g + prf) for g in range(40)]
    ctx = B.GroupContext(tables, **KINDS[kind])
    try:
        for mix in MIXES:
            check_list(torch, kind, ctx, tables, make_bins(mix, 40, rng), prf, rng)
    finally:
        ctx.close()
    sizes = GROUPED[kind][0] * 3
    tables = [random_table(n, 40, seed=100 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **KINDS[kind])
    try:
        for nbad in (0, 37):
            bins = rng.randint(0, len(sizes), size=500).astype(np.int32)
            bad_at = rng.choice(np.arange(2 * len(sizes), len(bins)), size=nbad, replace=False)
            bins[bad_at] = rng.choice([-1, -7, -2 ** 31, len(sizes), len(sizes) + 5, 2 ** 31 - 1], size=nbad)
            check_list(torch, kind, ctx, tables, bins, prf, rng)
    finally:
        ctx.close()
    sizes = GROUPED[kind][1]
    tables = [random_table(n, 24, seed=400 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, trimmed=True, **KINDS[kind])
    try:
        check_list(torch, kind, ctx, tables, rng.randint(0, len(sizes), size=600).astype(np.int32), prf, rng, trimmed=True)
    finally:
        ctx.close()
