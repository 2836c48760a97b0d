"""The restated layouts and the per-server bin reference the GPU tests compare every server's answer with
(tests/test_gpu_server_answers.py), checked on the host against the library's own placement: batchcode_ref.bins puts
every table row where b200dpf_batchcode_locate says, kwpir_ref.bins puts every item where b200dpf_kwpir_locate and the
placement rule say and leaves every other slot zero, and server_ref's answers equal a row-by-row restatement and
reconstruct the rows an end-to-end batch-code query wants.  No GPU needed."""
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

M64 = (1 << 64) - 1


def row_ids(n, e):
    """a table whose row r holds r and then columns derived from it: every copy names its row"""
    t = np.zeros((n, e), np.int32)
    t[:, 0] = np.arange(n)
    for c in range(1, e):
        t[:, c] = (np.arange(n, dtype=np.int64) * (2 * c + 1) + c).astype(np.int32)
    return t


@pytest.mark.parametrize("n,nbins", [(1, 1), (2, 1), (7, 3), (1000, 1), (1001, 7), (4099, 48), (20011, 48), (1537, 1536),
                                     (3001, 1536), (1536, 1536)])
def test_batchcode_bins_follow_locate(n, nbins):
    seed = (n * 0x9E3779B97F4A7C15 + nbins) & M64
    table = row_ids(n, 2)
    bins = BC.bins(table, n, nbins, seed)
    assert len(bins) == nbins
    for j in range(nbins):
        assert bins[j].shape == (3 * BC.per_copy(n, nbins, j), 2)
    assert sum(b.shape[0] for b in bins) == 3 * n
    seen = [np.zeros(b.shape[0], np.int32) for b in bins]
    for r in range(n):
        bs, rows = BC.locate(n, nbins, seed, r)
        for c in range(3):
            assert np.array_equal(bins[bs[c]][rows[c]], table[r]), (r, c)
            seen[bs[c]][rows[c]] += 1
    assert all((s == 1).all() for s in seen)


@pytest.mark.parametrize("n,expansion,e", [(1, 1.3, 1), (2, 1.3, 3), (100, 1.15, 14), (4097, 1.3, 16), (20000, 1.15, 1)])
def test_kwpir_bins_follow_locate(n, expansion, e):
    rng = np.random.RandomState(n)
    kw = np.unique(rng.randint(0, 1 << 63, 2 * n + 8, dtype=np.int64).astype(np.uint64) * np.uint64(3))[:n]
    kw[-1] = np.uint64(M64 - 1)                     # tag 2^64 - 1: both tag words all ones
    values = rng.randint(-2 ** 31, 2 ** 31, size=(n, e), dtype=np.int64).astype(np.int32)
    m = K.default_m(n, expansion)
    seed = 0xC0FFEE + n
    bins = K.bins(kw, values, m, seed)
    assert [b.shape for b in bins] == [(m, e + 2)] * 3
    where = B.kwpir_locate(m, seed, kw)
    assert np.array_equal(where, K.rows3(kw, m, seed))
    placed = np.zeros((3, m), bool)
    tag_of = {}
    for c in range(3):
        lo = bins[c][:, e].view(np.uint32).astype(np.uint64)
        hi = bins[c][:, e + 1].view(np.uint32).astype(np.uint64)
        for r in np.flatnonzero((lo | hi) != 0):
            tag_of[int(lo[r] | (hi[r] << np.uint64(32)))] = (c, int(r))
    assert len(tag_of) == n, "every item has exactly one slot"
    for i, w in enumerate(kw):
        c, r = tag_of[(int(w) + 1) & M64]
        assert r == where[i, c], "keyword %d is not in one of its three candidate rows" % i
        assert np.array_equal(bins[c][r, :e], values[i])
        placed[c, r] = True
    for c in range(3):
        assert not bins[c][~placed[c]].any(), "an empty slot is not all zeros"


def test_kwpir_bins_refuse_an_unfinished_placement():
    m = 100
    kw = np.arange(3 * m, dtype=np.uint64) * np.uint64(0x9E3779B1)
    assert K.place(kw, m, 7)[0] is None
    with pytest.raises(ValueError, match="does not finish"):
        K.bins(kw, np.zeros((3 * m, 1), np.int32), m, 7)


@pytest.mark.parametrize("kind", ["standard", "et", "xor"])
def test_bin_answers_equal_a_row_by_row_sum_and_reconstruct(kind):
    """the end-to-end batch-code case of test_batchcode_host.py: bins from the restated layout, keys from
    BatchCodeDPF.gen_queries, each server's answer from server_ref, equal to the answer summed row by row, and the
    pairs reconstruct the wanted rows"""
    torch = pytest.importorskip("torch")
    import dpf
    n, nbins, k, E, nq = 301, 12, 8, 3, 2
    seed = 0xABCDEF
    prf = dpf.DPF.PRF_CHACHA20
    rng = np.random.RandomState(7)
    table = rng.randint(-2 ** 31, 2 ** 31, size=(n, E), dtype=np.int64).astype(np.int32)
    d = dpf.BatchCodeDPF(prf, 0, nbins, seed=seed, early_termination=kind == "et", xor=kind == "xor")
    d.use_layout(n)
    bins = BC.bins(table, n, nbins, seed)
    assert [b.shape[0] for b in bins] == d.bin_sizes
    wanted = rng.randint(0, n, size=(nq, k)).astype(np.int64)
    qa, qb, slots = d.gen_queries(torch.as_tensor(wanted))
    out_a = S.query_answers(kind, prf, qa.numpy(), bins)
    out_b = S.query_answers(kind, prf, qb.numpy(), bins)
    ev = {"standard": B.eval_cpu, "et": B.eval_cpu_et, "xor": B.eval_cpu_xor}[kind]
    for q in range(nq):
        for g in range(nbins):
            for key, got in ((qa[q, g].numpy(), out_a[q, g]), (qb[q, g].numpy(), out_b[q, g])):
                share = ev(key, prf)
                if kind == "xor":
                    share = ((share.view(np.uint32)[:, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(-1)
                acc = np.zeros(E, np.uint32)
                for r in range(bins[g].shape[0]):
                    s = int(share[B.trimmed_alpha(r, bins[g].shape[0], S.SUFFIX[kind])]) & 0xFFFFFFFF
                    row = bins[g][r].view(np.uint32)
                    if kind == "xor":
                        acc ^= row if s else np.uint32(0)
                    else:
                        acc = ((acc.astype(np.uint64) + np.uint64(s) * row.astype(np.uint64)) & 0xFFFFFFFF).astype(np.uint32)
                assert np.array_equal(got.view(np.uint32), acc), (q, g)
    rows, found = d.reconstruct(torch.as_tensor(out_a), torch.as_tensor(out_b), slots)
    assert found.numpy().mean() > 0.5
    for q in range(nq):
        for i in range(k):
            if found[q, i]:
                assert np.array_equal(rows[q, i].numpy(), table[wanted[q, i]]), (q, i)


@pytest.mark.parametrize("kind", ["standard", "et", "xor"])
def test_compact_queries_unpack_to_their_keys(kind):
    """server_ref.unpack_queries inverts GroupContext.pack_queries' layout, for trimmed bins of several depths"""
    s = S.SUFFIX[kind]
    sizes = [1, 5, 300, 3001]
    rng = np.random.RandomState(3)
    keys = np.zeros((2, len(sizes), B.KEY_WORDS), np.int32)
    packed = []
    for q in range(2):
        parts = []
        for g, rows in enumerate(sizes):
            a, _ = PM.gen_keys(kind, S.domain(rows, kind), [B.trimmed_alpha(int(rng.randint(0, rows)), rows, s)], B.PRF_AES128, q * 10 + g)
            keys[q, g] = a[0]
            parts.append(np.frombuffer(getattr(B, "key_pack" + s)(a[0]), np.uint8))
        packed.append(np.concatenate(parts))
    assert np.array_equal(S.unpack_queries(kind, sizes, np.stack(packed)), keys)


def test_edge_rows():
    for kind in ("standard", "et", "xor"):
        for rows, trimmed in ((1, True), (3001, True), (1024, False), (256, False)):
            r = S.edge_rows(rows, kind, trimmed)
            assert r[0] == 0 and r[1] == rows - 1 and all(0 <= x < rows for x in r)
    idx = S.key_index(1024, "standard", False)
    assert idx[S.edge_rows(1024, "standard", False)[2]] == 0x155 and idx[S.edge_rows(1024, "standard", False)[3]] == 0x2AA
