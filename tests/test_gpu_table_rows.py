"""Tables that span several of the 64 MiB stages through which a context's create carries the caller's rows to the
device, for every kind of key and every create path: plain contexts whole and in 2 and 4 entry-range shards, trimmed,
grouped (bins of powers of two and trimmed bins), batch-code and keyword-PIR contexts.  Each is created from pageable
host, pinned host and device memory.

At E = 4096 a stage holds 4,096 rows (4,098 values of 4,094 columns on a keyword-PIR context), so every table below
crosses at least three stage boundaries, and those whose size is free end in a partial stage.  Keys target the first
and last row of every stage (of a shard's own rows on a shard).  One server's results are compared bit for bit with
the exact reference of tests/wide_oracle.py over the whole table, which catches a row written to the wrong place
anywhere in it, and every pair must reconstruct its row."""
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
import kwpir_ref as K  # noqa: E402
import plan_matrix as PM  # noqa: E402
import wide_oracle as W  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

E = 4096
STAGE_BYTES = 64 << 20
CHUNK = STAGE_BYTES // (4 * E)          # 4,096 rows per stage
N = 1 << 16                              # plain tables: 16, 8 and 4 stages per shard of 1, 2 and 4
RAGGED = 3 * CHUNK + 1000                # trimmed tables, the largest trimmed bin and the batch-code table
KW_E = 4094
KW_CHUNK = STAGE_BYTES // (4 * KW_E)     # 4,098 values per stage
KW_N = 3 * KW_CHUNK + 1000
SOURCES = ("pageable", "pinned", "device")
SUFFIX = {"standard": "", "et": "_et", "xor": "_xor"}
PRF = {"standard": B.PRF_AES128, "et": B.PRF_CHACHA20, "xor": B.PRF_SALSA20}


@pytest.fixture(scope="module")
def table():
    """(the [N, E] table in pageable memory, {source: the address of the same bytes there})"""
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    host = np.random.default_rng(5).integers(0, 2**32, size=(N, E), dtype=np.uint32).view(np.int32)
    pinned = torch.from_numpy(host).pin_memory()
    device = pinned.cuda()
    torch.cuda.synchronize()
    yield host, {"pageable": host.ctypes.data, "pinned": pinned.data_ptr(), "device": device.data_ptr()}
    W.clear_cache()


def edges(rows, chunk):
    """the first and last of every run of `chunk` rows in [0, rows)"""
    return sorted({r for c0 in range(0, rows, chunk) for r in (c0, min(c0 + chunk, rows) - 1)})


def handle_of(cls, entry_size, create, name):
    ctx = cls.__new__(cls)
    ctx.entry_size = entry_size
    ctx.handle = C.c_void_p()
    B._check(create(C.byref(ctx.handle)), name)
    return ctx


def trimmed_keys(kind, n, rows, prf, seed):
    """keys of both servers for rows `rows` of a trimmed table of n rows"""
    alphas = [B.trimmed_alpha(int(r), n, SUFFIX[kind]) for r in rows]
    return PM.gen_keys(kind, B.trimmed_domain(n, SUFFIX[kind]), alphas, prf, seed=seed)


def trimmed_expected(kind, prf, keys, t):
    """the result of `keys` on a trimmed table t: the reference on t's rows placed at their key indices"""
    n = t.shape[0]
    at = np.zeros((B.trimmed_domain(n, SUFFIX[kind]), t.shape[1]), np.int32)
    at[[B.trimmed_alpha(r, n, SUFFIX[kind]) for r in range(n)]] = t
    return W.expected(kind, prf, keys, at)


def combine(kind, parts):
    out = np.zeros_like(parts[0]).view(np.uint32)
    for p in parts:
        out = out ^ p.view(np.uint32) if kind == "xor" else out + p.view(np.uint32)
    return out.view(np.int32)


@pytest.mark.parametrize("shards", (1, 2, 4))
@pytest.mark.parametrize("kind", PM.KINDS)
def test_plain(table, kind, shards):
    host, addr = table
    prf = PRF[kind]
    alphas = []
    for r in range(shards):
        own = np.flatnonzero(PM.owned_rows(kind, N, r, shards))
        alphas += [int(own[j]) for j in edges(len(own), CHUNK)]
    a, b = PM.gen_keys(kind, N, alphas, prf, seed=shards)
    want = [W.expected(kind, prf, a, host, r, shards) for r in range(shards)]
    for src in SOURCES:
        ra, rb = [], []
        for r in range(shards):
            name = "b200dpf_create" + SUFFIX[kind]
            ctx = handle_of(B.Context, E, lambda h: getattr(B.lib(), name)(h, C.c_void_p(addr[src]), N, E, 0, r, shards), name)
            try:
                ra.append(ctx.eval(a, prf))
                rb.append(ctx.eval(b, prf))
            finally:
                ctx.close()
            assert np.array_equal(ra[-1], want[r]), "%s, shard %d of %d" % (src, r, shards)
        assert np.array_equal(PM.reconstruct(kind, combine(kind, ra), combine(kind, rb)), host[alphas]), src


@pytest.mark.parametrize("kind", PM.KINDS)
def test_trimmed(table, kind):
    host, addr = table
    prf, t, rows = PRF[kind], host[:RAGGED], edges(RAGGED, CHUNK)
    a, b = trimmed_keys(kind, RAGGED, rows, prf, seed=1)
    want = trimmed_expected(kind, prf, a, t)
    for src in SOURCES:
        ctx = handle_of(B.Context, E, lambda h: B.lib().b200dpf_create_trimmed(h, C.c_void_p(addr[src]), RAGGED, E, 0,
                                                                                  B.KIND_IDS[SUFFIX[kind]]),
                        "b200dpf_create_trimmed")
        try:
            ra, rb = ctx.eval(a, prf), ctx.eval(b, prf)
        finally:
            ctx.close()
        assert np.array_equal(ra, want), src
        assert np.array_equal(PM.reconstruct(kind, ra, rb), t[rows]), src


def check_grouped(kind, prf, make, bins, trimmed):
    """Create a grouped context three times by make(source), whose bins hold the host tables `bins`, and evaluate keys
    for the rows targets[g] of each bin g: every result against the reference, every pair against its row."""
    keys_a, keys_b, ids, want, rows = [], [], [], [], []
    for g, (t, targets) in enumerate(bins):
        if not targets:
            continue
        if trimmed:
            a, b = trimmed_keys(kind, t.shape[0], targets, prf, seed=g)
            want.append(trimmed_expected(kind, prf, a, t))
        else:
            a, b = PM.gen_keys(kind, t.shape[0], targets, prf, seed=g)
            want.append(W.expected(kind, prf, a, t))
        keys_a.append(a)
        keys_b.append(b)
        ids += [g] * len(targets)
        rows.append(t[targets])
    a, b, ids, want, rows = (np.concatenate(x) for x in (keys_a, keys_b, [ids], want, rows))
    for src in SOURCES:
        ctx = make(src)
        try:
            ra, rb = ctx.eval(a, ids, prf), ctx.eval(b, ids, prf)
        finally:
            ctx.close()
        assert np.array_equal(ra, want), src
        assert np.array_equal(PM.reconstruct(kind, ra, rb), rows), src


@pytest.mark.parametrize("trimmed", (False, True), ids=("pow2", "trimmed"))
@pytest.mark.parametrize("kind", PM.KINDS)
def test_grouped(table, kind, trimmed):
    """bins at several offsets of the table: the first spans four stages (trimmed: three and a partial one)"""
    host, addr = table
    spans = [(0, RAGGED), (20000, 700), (30000, 5000)] if trimmed else [(0, 1 << 14), (20000, 1 << 13), (40000, 256)]
    sizes = np.array([s for _, s in spans], np.int64)

    def make(src):
        ptrs = (C.c_void_p * len(spans))(*[addr[src] + o * E * 4 for o, _ in spans])
        if trimmed:
            return handle_of(B.GroupContext, E, lambda h: B.lib().b200dpf_group_create_trimmed(
                h, ptrs, sizes, len(spans), E, 0, B.KIND_IDS[SUFFIX[kind]]), "b200dpf_group_create_trimmed")
        name = "b200dpf_group_create" + SUFFIX[kind]
        return handle_of(B.GroupContext, E, lambda h: getattr(B.lib(), name)(h, ptrs, sizes, len(spans), E, 0), name)

    check_grouped(kind, PRF[kind], make, [(host[o:o + s], edges(s, CHUNK)) for o, s in spans], trimmed)


@pytest.mark.parametrize("kind", PM.KINDS)
def test_batchcode(table, kind):
    """a RAGGED-row table as a batch code of 4 bins: the keys target every copy of the first and last row of each stage"""
    host, addr = table
    nbins, seed, t = 4, 11, host[:RAGGED]
    m = [(RAGGED - j + nbins - 1) // nbins for j in range(nbins)]
    bins = [np.zeros((3 * m[j], E), np.int32) for j in range(nbins)]
    wanted = set(edges(RAGGED, CHUNK))
    targets = [[] for _ in range(nbins)]
    for r in range(RAGGED):
        bs, rs = B.batchcode_locate(RAGGED, nbins, seed, r)
        for j, row in zip(bs, rs):
            bins[j][row] = t[r]
            if r in wanted:
                targets[j].append(int(row))

    def make(src):
        return handle_of(B.BatchCodeContext, E, lambda h: B.lib().b200dpf_batchcode_create(
            h, C.c_void_p(addr[src]), RAGGED, E, nbins, seed, 0, B.KIND_IDS[SUFFIX[kind]]), "b200dpf_batchcode_create")

    check_grouped(kind, PRF[kind], make, list(zip(bins, targets)), True)


@pytest.mark.parametrize("kind", PM.KINDS)
def test_kwpir(table, kind):
    """KW_N values of the widest size a keyword-PIR context takes, read from the table's bytes; keywords stay on the
    host.  The keys target the slots of the first and last item of each stage."""
    host, addr = table
    values = host.reshape(-1)[:KW_N * KW_E].reshape(KW_N, KW_E)
    keywords = np.random.default_rng(7).integers(0, 2**63, size=KW_N, dtype=np.uint64)
    assert len(np.unique(keywords)) == KW_N
    m, seed = K.default_m(KW_N), 3
    rounds, owner = K.place(keywords, m, seed)
    assert rounds is not None
    tag = K.tags(keywords, owner, m).reshape(-1)
    rows = np.zeros((3 * m, KW_E + 2), np.int32)
    full = owner >= 0
    rows[full, :KW_E] = values[owner[full]]
    rows[:, KW_E] = (tag & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.int32)
    rows[:, KW_E + 1] = (tag >> np.uint64(32)).astype(np.uint32).view(np.int32)
    slots = [int(np.flatnonzero(owner == i)[0]) for i in edges(KW_N, KW_CHUNK)]
    bins = [(rows[c * m:(c + 1) * m], sorted(s - c * m for s in slots if s // m == c)) for c in range(3)]

    def make(src):
        return handle_of(B.KeywordContext, KW_E + 2, lambda h: B.lib().b200dpf_kwpir_create(
            h, keywords.ctypes.data_as(C.c_void_p), C.c_void_p(addr[src]), KW_N, KW_E, m, seed, 0, B.KIND_IDS[SUFFIX[kind]]),
            "b200dpf_kwpir_create")

    check_grouped(kind, PRF[kind], make, bins, True)
