"""Entries up to the documented 4096 columns (include/b200dpf.h: entry_size 1 .. 4096) on the GPU, for every kind
of key, on plain and grouped contexts.  Every result is compared bit for bit with an exact reference that never
comes from the GPU (tests/wide_oracle.py), and every pair reconstructs its row.  One server's result against the
reference is what catches a planning error: both servers hold the same share at every row but alpha, so a
skipped slice, a dropped column or a chunk written at the wrong offset cancels out of a - b (or a ^ b).

  * test_plain: E from 255 to 4096 (4033 leaves one column in the last 64-column slice), batches of 1 to 100
    keys, each of the defaults, leaf_cache=0, mac_tma=0, leaf_cache_mb=1 (chunks of 64 keys at n = 2^12, and at
    n = 2^14 one key group over the cap) and one_launch=0 on one live context, through eval, eval_packed,
    eval_gather, eval_device and eval_device(accumulate=True); the launch count proves which path ran;
  * test_shards: the 2 and 4 entry-range shards of a 4096-column table combine to the whole table's result;
  * test_extremes: whole columns and rows of INT32_MIN, INT32_MAX and -1 at 4096 columns;
  * test_update_rows: row updates at 4095 columns (single-word copies) and 4096 (16-byte copies), on the host
    and device paths of a plain context and on a grouped context;
  * test_grouped: grouped contexts at 255, 1000 and 4096 columns, host and device evaluations and query
    batches of wire keys and compact queries;
  * test_python_surfaces: dpf.DPF of each kind and dpf.BinnedDPF on 4096-column torch tables."""
import os
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402
import plan_matrix as PM  # noqa: E402
import wide_oracle as W  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

D, S, C, A = B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128
I32_MIN, I32_MAX = -2**31, 2**31 - 1
SUFFIX = {"standard": "", "et": "_et", "xor": "_xor"}
ENTRIES = ("eval", "eval_packed", "eval_gather", "eval_device")
# columns per pass of a fused evaluation without the leaf cache: 4 * the widest row vector the kind's kernel takes
UNCACHED_COLS = {"standard": 64, "et": 32, "xor": 16}
DEFAULTS = {"leaf_cache": 1, "leaf_cache_mb": 16384, "mac_tma": 1, "one_launch": 1}
OPTION_ROWS = [{}, {"leaf_cache": 0}, {"mac_tma": 0}, {"leaf_cache_mb": 1}, {"one_launch": 0}]


@pytest.fixture(scope="module", autouse=True)
def wall_time(request):
    """print the module's wall time: most of it is the host reference"""
    t0 = time.perf_counter()
    yield
    W.clear_cache()
    capture = request.config.pluginmanager.get_plugin("capturemanager")
    with capture.global_and_fixture_disabled():
        print("\ntest_gpu_wide_entries.py: %.1f s wall" % (time.perf_counter() - t0))


@pytest.fixture(scope="module", autouse=True)
def cuda_device():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")


def wide_table(n, e, seed):
    return np.random.default_rng(seed).integers(0, 2**32, size=(n, e), dtype=np.uint32).view(np.int32)


def alphas_for(n, batch, seed):
    al = np.random.RandomState(seed).randint(0, n, size=batch).astype(np.int64)
    al[:min(batch, 3)] = [0, n - 1, n // 2 + 1][:min(batch, 3)]
    return al


def context(kind, table, shard_rank=0, shard_count=1):
    return B.Context(table, shard_rank=shard_rank, shard_count=shard_count, early_termination=kind == "et",
                     xor=kind == "xor")


def set_options(ctx, row):
    for name, value in dict(DEFAULTS, **row).items():
        ctx.set_option(name, value)


def device_out(base):
    return torch.from_numpy(np.ascontiguousarray(base)).cuda()


def evaluate(ctx, kind, entry, keys, prf):
    """results of `keys` through entry point `entry`; eval_device writes into a buffer of -1"""
    if entry == "eval":
        return ctx.eval(keys, prf)
    if entry == "eval_packed":
        pack = getattr(B, "key_pack" + SUFFIX[kind])
        return ctx.eval_packed(b"".join(pack(k) for k in keys), len(keys), prf)
    if entry == "eval_gather":
        return ctx.eval_gather(list(keys), prf)
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys)).cuda()
    out = torch.full((len(keys), ctx.entry_size), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.eval_device(keys_dev.data_ptr(), len(keys), prf, out.data_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy()


def accumulate(ctx, keys, prf, base):
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys)).cuda()
    out = device_out(base)
    torch.cuda.synchronize()
    ctx.eval_device(keys_dev.data_ptr(), len(keys), prf, out.data_ptr(), accumulate=True)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def acc_ref(kind, base, res):
    b, r = base.view(np.uint32), res.view(np.uint32)
    return (b ^ r if kind == "xor" else b + r).view(np.int32)


def plain_launches(kind, n_local, e, batch, row):
    """(launches, chunks) of one evaluation on a plain context, e > 32, with the cooperative launch (run_pipeline
    and launch_plan): keys in chunks whose leaf cache fits leaf_cache_mb; a chunk of >= 17 keys with the cache
    is one fused pass and a MAC pass per 64-column slice, any other one fused pass per UNCACHED_COLS columns.
    one_launch=0 may add a frontier launch per chunk."""
    o = dict(DEFAULTS, **row)
    per_group = 32 * n_local * 4
    cap = o["leaf_cache_mb"] << 20
    cached = kind != "xor" and o["leaf_cache"] and batch >= 17 and per_group <= cap
    chunk = max(1, cap // per_group) * 32 if cached else batch
    total = chunks = 0
    for k0 in range(0, batch, chunk):
        m = min(chunk, batch - k0)
        total += 1 + -(-e // 64) if cached and m >= 17 else -(-e // UNCACHED_COLS[kind])
        chunks += 1
    return total, chunks


def check_launches(ctx, kind, e, batch, row, where, n_local=None):
    want, chunks = plain_launches(kind, ctx.n if n_local is None else n_local, e, batch, row)
    got = ctx.last_launches
    if dict(DEFAULTS, **row)["one_launch"]:
        assert got == want, "%s: %d launches, expected %d" % (where, got, want)
    else:
        assert want <= got <= want + chunks, "%s: %d launches, expected %d to %d" % (where, got, want, want + chunks)


def shape_id(kind, shape):
    prf, n, e, batch = shape
    return "%s-%s-n%d-E%d-B%d" % (kind, B.PRF_NAMES[prf], n, e, batch)


# (prf, n, E, batch): each kind meets every PRF and every entry size; batches of 1 to 3 (XOR-shared key quads
# padded), 16 (no leaf cache), 17 and 33 (one cached chunk), 100 (at n = 2^12 with leaf_cache_mb = 1: chunks of
# 64 and 36 keys; at n = 2^14: one key group over the cap)
PLAIN = {
    "standard": [(D, 1 << 12, 255, 17), (S, 1 << 12, 256, 100), (C, 1 << 10, 257, 3), (A, 1 << 14, 1000, 33),
                 (D, 1 << 14, 4033, 16), (S, 1 << 12, 4095, 100), (C, 1 << 14, 4096, 100), (A, 1 << 12, 4096, 1)],
    "et": [(S, 1 << 12, 255, 100), (C, 1 << 12, 256, 16), (A, 1 << 10, 257, 17), (D, 1 << 14, 1000, 1),
           (S, 1 << 14, 4033, 33), (C, 1 << 12, 4095, 100), (A, 1 << 14, 4096, 100), (D, 1 << 12, 4096, 3)],
    "xor": [(A, 256, 255, 1), (D, 1 << 12, 256, 3), (S, 1 << 12, 257, 16), (C, 1 << 14, 1000, 17),
            (A, 1 << 12, 4033, 33), (D, 1 << 14, 4095, 3), (S, 1 << 14, 4096, 33), (C, 1 << 12, 4096, 100)],
}
PLAIN_CASES = [(k, s) for k in PM.KINDS for s in PLAIN[k]]


@pytest.mark.parametrize("kind,shape", PLAIN_CASES, ids=[shape_id(k, s) for k, s in PLAIN_CASES])
def test_plain(kind, shape):
    prf, n, e, batch = shape
    table = wide_table(n, e, seed=e + batch)
    alphas = alphas_for(n, batch, seed=e)
    a, b = PM.gen_keys(kind, n, alphas, prf, seed=n + e)
    want = W.expected(kind, prf, a, table)
    base = wide_table(batch, e, seed=7 * e)
    ctx = context(kind, table)
    try:
        rb = ctx.eval(b, prf)
        assert np.array_equal(PM.reconstruct(kind, want, rb), table[alphas]), "%s: pairs" % shape_id(kind, shape)
        for row in OPTION_ROWS:              # one live context: every plan follows another
            set_options(ctx, row)
            for entry in ENTRIES:
                where = "%s %s %s" % (shape_id(kind, shape), row, entry)
                assert np.array_equal(evaluate(ctx, kind, entry, a, prf), want), where
                check_launches(ctx, kind, e, batch, row, where)
            where = "%s %s eval_device accumulate" % (shape_id(kind, shape), row)
            assert np.array_equal(accumulate(ctx, a, prf, base), acc_ref(kind, base, want)), where
            check_launches(ctx, kind, e, batch, row, where)
    finally:
        ctx.close()


@pytest.mark.parametrize("kind,prf", [("standard", A), ("et", D), ("xor", C)])
def test_shards(kind, prf):
    n, e, batch = 1 << 14, 4096, 20
    table = wide_table(n, e, seed=prf)
    alphas = alphas_for(n, batch, seed=prf)
    a, _ = PM.gen_keys(kind, n, alphas, prf, seed=prf)
    whole = W.expected(kind, prf, a, table)
    for g in (2, 4):
        parts = []
        for r in range(g):
            ctx = context(kind, table, r, g)
            try:
                got = ctx.eval(a, prf)
                where = "%s shard %d/%d" % (kind, r, g)
                check_launches(ctx, kind, e, batch, {}, where, n_local=n // g)
            finally:
                ctx.close()
            assert np.array_equal(got, W.expected(kind, prf, a, table, r, g)), where
            parts.append(got)
        assert np.array_equal(PM.combine(kind, parts), whole), "%s: %d shards combined" % (kind, g)


EXTREMES = (I32_MIN, I32_MAX, -1)


@pytest.mark.parametrize("kind,prf", [("standard", S), ("et", A), ("xor", D)])
def test_extremes(kind, prf):
    """columns and rows of INT32_MIN, INT32_MAX and -1 at both ends of a 2^14 x 4096 table: every column sum
    wraps many times"""
    n, e, batch = 1 << 14, 4096, 33
    table = wide_table(n, e, seed=11 + prf)
    for j, v in enumerate(EXTREMES):
        table[:, [j, 16 + j, 2046 + j, 4033 + j, e - 3 + j]] = v
        table[[j, n - 3 + j]] = v
    alphas = alphas_for(n, batch, seed=12)
    alphas[3:6] = [1, 2, n - 3]
    a, b = PM.gen_keys(kind, n, alphas, prf, seed=13)
    want = W.expected(kind, prf, a, table)
    ctx = context(kind, table)
    try:
        assert np.array_equal(PM.reconstruct(kind, want, ctx.eval(b, prf)), table[alphas])
        for row in ({}, {"leaf_cache": 0}, {"mac_tma": 0}):
            set_options(ctx, row)
            assert np.array_equal(ctx.eval(a, prf), want), "%s %s" % (kind, row)
            check_launches(ctx, kind, e, batch, row, "%s %s" % (kind, row))
    finally:
        ctx.close()


def apply_updates(table, indices, rows):
    """table[indices[j]] := rows[j] in order (the last occurrence wins); indices outside [0, n) skipped"""
    for i, r in zip(indices, rows):
        if 0 <= i < len(table):
            table[i] = r


GROUP_KINDS = {      # GroupContext keyword, bin sizes (the smallest each kind takes, up to 2^14)
    "standard": ({}, [2, 64, 1 << 10, 1 << 12, 1 << 14]),
    "et": ({"early_termination": True}, [8, 64, 1 << 10, 1 << 12, 1 << 14]),
    "xor": ({"xor": True}, [256, 512, 1 << 10, 1 << 12, 1 << 14]),
}
UPDATE_CASES = [(k, e) for k in PM.KINDS for e in (4095, 4096)]


@pytest.mark.parametrize("kind,e", UPDATE_CASES, ids=["%s-E%d" % c for c in UPDATE_CASES])
def test_update_rows(kind, e):
    prf = {"standard": C, "et": S, "xor": A}[kind]
    n, batch = 1 << 12, 33
    table = wide_table(n, e, seed=e)
    alphas = alphas_for(n, batch, seed=e)
    alphas[3:5] = [5, 77]
    a, b = PM.gen_keys(kind, n, alphas, prf, seed=e)
    ctx = context(kind, table)
    try:
        assert np.array_equal(ctx.eval(a, prf), W.expected(kind, prf, a, table)), "before the updates"
        # host path: the first and last rows, repeated indices (the last one wins)
        idx = np.array([0, n - 1, 5, 5, 77, 0, 77, 77, 1], np.int64)
        rows = wide_table(len(idx), e, seed=e + 1)
        rows[1] = I32_MIN
        ctx.update_rows(idx, rows)
        apply_updates(table, idx, rows)
        # an index out of range on the host path: refused, nothing applied
        with pytest.raises(B.B200DPFError, match=r"index %d out of range \[0, %d\)" % (n, n)):
            ctx.update_rows(np.array([3, n], np.int64), wide_table(2, e, seed=e + 2))
        # device path: out-of-range indices skipped, repeated ones (the last one wins), first and last rows
        idx_d = np.array([n - 1, -1, 9, n, 9, 1 << 40, 0, n - 1, 2, -(1 << 40)], np.int64)
        rows_d = wide_table(len(idx_d), e, seed=e + 3)
        rows_d[7] = I32_MAX
        idx_dev, rows_dev = torch.from_numpy(idx_d).cuda(), torch.from_numpy(rows_d).cuda()
        torch.cuda.synchronize()
        ctx.update_rows_device(idx_dev.data_ptr(), rows_dev.data_ptr(), len(idx_d),
                               torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        apply_updates(table, idx_d, rows_d)
        want = W.expected(kind, prf, a, table)
        assert np.array_equal(PM.reconstruct(kind, want, ctx.eval(b, prf)), table[alphas])
        for row in ({}, {"leaf_cache": 0}):
            set_options(ctx, row)
            assert np.array_equal(ctx.eval(a, prf), want), "%s after the updates" % row
            assert np.array_equal(evaluate(ctx, kind, "eval_device", a, prf), want), "%s after the updates" % row
    finally:
        ctx.close()

    # a grouped context: its rows are padded to 16 columns, not 64
    kw, sizes = GROUP_KINDS[kind]
    sizes = sizes[1:4]
    tables = [wide_table(m, e, seed=e + 10 + g) for g, m in enumerate(sizes)]
    ka, kb, bins, galphas = gen_pairs(kind, sizes, [5, 17, 33], prf, seed=e)
    ctx = B.GroupContext(tables, **kw)
    try:
        ub = np.array([0, 0, 1, 2, 2, 1, 0, 2], np.int32)
        ui = np.array([0, sizes[0] - 1, 0, sizes[2] - 1, 3, 0, 0, sizes[2] - 1], np.int64)
        urows = wide_table(len(ub), e, seed=e + 4)
        ctx.update_rows(ub, ui, urows)
        for g, i, r in zip(ub, ui, urows):
            tables[g][i] = r
        check_group(kind, ctx, tables, ka, kb, bins, galphas, prf, "%s E=%d grouped, updated" % (kind, e))
    finally:
        ctx.close()


def gen_keys(kind, alphas, n, prf, rng):
    if kind == "standard":
        return B.gen_batch(alphas, n, rng.randint(0, 2**31, size=len(alphas)), prf)
    seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
    return (B.gen_batch_et if kind == "et" else B.gen_batch_xor)(alphas, n, seeds, prf)


def gen_pairs(kind, sizes, per_bin, prf, seed):
    """shuffled (bin, key) pairs: key pairs of every bin (its first and last row among the targets)"""
    rng = np.random.RandomState(seed)
    ka, kb, bins, alphas = [], [], [], []
    for g, (n, cnt) in enumerate(zip(sizes, per_bin)):
        al = rng.randint(0, n, size=cnt).astype(np.int64)
        al[:2] = [0, n - 1][:cnt]
        a, b = gen_keys(kind, al, n, prf, rng)
        ka.append(a); kb.append(b); bins += [g] * cnt; alphas.append(al)
    order = rng.permutation(len(bins))
    return (np.concatenate(ka)[order], np.concatenate(kb)[order], np.array(bins, np.int32)[order],
            np.concatenate(alphas)[order])


def group_expected(kind, prf, keys, bins, tables):
    """each key's reference on its own bin"""
    out = np.zeros((len(keys), tables[0].shape[1]), np.int32)
    for g, t in enumerate(tables):
        sel = np.nonzero(bins == g)[0]
        if len(sel):
            out[sel] = W.expected(kind, prf, keys[sel], t)
    return out


def group_device(ctx, keys, bins, prf):
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys)).cuda()
    out = torch.full((len(keys), ctx.entry_size), -1, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream()
    torch.cuda.synchronize()
    ctx.eval_device(keys_dev.data_ptr(), bins, prf, out.data_ptr(), st.cuda_stream)
    st.synchronize()
    return out.cpu().numpy()


def check_group(kind, ctx, tables, ka, kb, bins, alphas, prf, where):
    """host and device evaluations of ka against the reference, and the pairs reconstruct their rows"""
    want = group_expected(kind, prf, ka, bins, tables)
    passes = -(-ctx.entry_size // 16)
    assert np.array_equal(ctx.eval(ka, bins, prf), want), where + ": eval"
    assert np.array_equal(group_device(ctx, ka, bins, prf), want), where + ": eval_device"
    assert ctx.last_launches == passes, "%s: %d launches, expected %d" % (where, ctx.last_launches, passes)
    rb = group_device(ctx, kb, bins, prf)
    rows = np.stack([tables[g][al] for g, al in zip(bins, alphas)])
    assert np.array_equal(PM.reconstruct(kind, want, rb), rows), where + ": pairs"


GROUP_CASES = [(k, e, int(prf)) for i, k in enumerate(PM.KINDS)
               for e, prf in zip((255, 1000, 4096), np.roll((D, S, C, A), -i))]
PER_BIN = [1, 3, 5, 33, 70]           # partial key groups, and more than one 32-key group in two bins


@pytest.mark.parametrize("kind,e,prf", GROUP_CASES,
                         ids=["%s-E%d-%s" % (k, e, B.PRF_NAMES[p]) for k, e, p in GROUP_CASES])
def test_grouped(kind, e, prf):
    kw, sizes = GROUP_KINDS[kind]
    ka, kb, bins, alphas = gen_pairs(kind, sizes, PER_BIN, prf, seed=e)
    tables = [wide_table(m, e, seed=e + g) for g, m in enumerate(sizes)]
    ctx = B.GroupContext(tables, **kw)
    try:
        where = "%s E=%d %s" % (kind, e, B.PRF_NAMES[prf])
        check_group(kind, ctx, tables, ka, kb, bins, alphas, prf, where)
        # query batches: one key per bin per query, each bin's first and last row among the targets
        nq, nbins = 3, len(sizes)
        rng = np.random.RandomState(e + 1)
        qa = np.zeros((nq, nbins, B.KEY_WORDS), np.int32)
        qb = np.zeros_like(qa)
        qal = np.zeros((nq, nbins), np.int64)
        for g, m in enumerate(sizes):
            qal[:, g] = [0, m - 1, rng.randint(0, m)]
            qa[:, g], qb[:, g] = gen_keys(kind, qal[:, g], m, prf, rng)
        want = np.stack([W.expected(kind, prf, qa[:, g], tables[g]) for g in range(nbins)], axis=1)
        rows = np.stack([np.stack([tables[g][al] for g, al in enumerate(r)]) for r in qal])
        for compact in (False, True):
            got = {}
            for side, keys in (("a", qa), ("b", qb)):
                keys_dev = torch.from_numpy(ctx.pack_queries(keys) if compact else keys).cuda()
                out = torch.full((nq, nbins, e), -1, dtype=torch.int32, device="cuda")
                torch.cuda.synchronize()
                ctx.eval_queries_device(keys_dev.data_ptr(), nq, prf, out.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream, compact=compact)
                torch.cuda.synchronize()
                got[side] = out.cpu().numpy()
            what = "%s: queries%s" % (where, " compact" if compact else "")
            assert np.array_equal(got["a"], want), what
            assert ctx.last_launches == -(-e // 16), what
            assert np.array_equal(PM.reconstruct(kind, got["a"], got["b"]), rows), what + ": pairs"
    finally:
        ctx.close()


@pytest.mark.parametrize("kind,prf", [("standard", D), ("et", S), ("xor", C)])
def test_python_surfaces(kind, prf):
    import dpf
    n, e, batch = 1 << 12, 4096, 20
    table = wide_table(n, e, seed=31 + prf)
    alphas = alphas_for(n, batch, seed=32)
    a, b = PM.gen_keys(kind, n, alphas, prf, seed=33)
    want = W.expected(kind, prf, a, table)
    d = dpf.DPF(prf=prf, early_termination=kind == "et", xor=kind == "xor")
    try:
        d.eval_init(torch.from_numpy(table))
        assert np.array_equal(d.eval_gpu(torch.from_numpy(a)).numpy(), want), kind + ": tensor keys"
        assert np.array_equal(d.eval_gpu([torch.from_numpy(k) for k in a]).numpy(), want), kind + ": key list"
        rb = d.eval_gpu(torch.from_numpy(b)).numpy()
        assert np.array_equal(PM.reconstruct(kind, want, rb), table[alphas])
    finally:
        d.close()
    if kind != "standard":
        return
    sizes = [2, 64, 1 << 10, 1 << 12]
    tables = [wide_table(m, e, seed=40 + g) for g, m in enumerate(sizes)]
    ka, kb, bins, galphas = gen_pairs(kind, sizes, [3, 5, 17, 33], prf, seed=41)
    want = group_expected(kind, prf, ka, bins, tables)
    bd = dpf.BinnedDPF(prf=prf)
    try:
        bd.eval_init([torch.from_numpy(t) for t in tables])
        assert np.array_equal(bd.eval_gpu(torch.from_numpy(ka), bins).numpy(), want), "BinnedDPF"
        rb = bd.eval_gpu(torch.from_numpy(kb), bins).numpy()
        assert np.array_equal(PM.reconstruct(kind, want, rb), np.stack([tables[g][al] for g, al in zip(bins, galphas)]))
    finally:
        bd.close()
