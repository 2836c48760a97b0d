"""Every plan the tuning options select gives the same result (include/b200dpf.h: "Results never depend on
them"), for every kind of key, bit-exact against references that never come from the GPU (tests/plan_matrix.py):

  * test_option_pairs: every pair of levels of every two options (a pairwise covering array), run back to
    back on one live context per shape and shard, through every host and device entry point;
  * test_tree_top: every tree-top item size, balanced or not, in one launch or several, with more key
    groups than blocks (the one-launch kernel's host-quota branch) and on sparse tables at n = 2^20;
  * test_work_item_sizes: every work-item size up to 16 levels, with and without the frontier, up to
    n = 2^24 (AES: the deepest pending-sibling stacks, split around the T-tables);
  * test_accumulate: b200dpf_eval_device_acc on every path that clears the result otherwise, and shard
    contexts adding their partials into one buffer."""
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
import plan_matrix as PM  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

D, S, C, A = B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128
SUFFIX = {"standard": "", "et": "_et", "xor": "_xor"}
ENTRIES = ("eval", "eval_packed", "eval_gather", "eval_device")


def context(kind, table, shard_rank=0, shard_count=1):
    return B.Context(table, shard_rank=shard_rank, shard_count=shard_count, early_termination=kind == "et",
                     xor=kind == "xor")


def set_options(ctx, row):
    for name, value in row.items():
        ctx.set_option(name, value)


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


def expand(ctx, kind, keys, prf):
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys)).cuda()
    width = ctx.n // 32 if kind == "xor" else ctx.n
    out = torch.full((len(keys), width), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.expand_device(keys_dev.data_ptr(), len(keys), prf, out.data_ptr())
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    return got.view(np.uint32) if kind == "xor" else got


def alphas_for(n, batch, seed):
    al = np.random.RandomState(seed).randint(0, n, size=batch).astype(np.int64)
    al[:min(batch, 3)] = [0, n - 1, n // 2 + 1][:min(batch, 3)]
    return al


def shape_id(kind, shape):
    prf, n, e, batch, g = shape
    return "%s-%s-n%d-E%d-B%d-G%d" % (kind, B.PRF_NAMES[prf], n, e, batch, g)


# (prf, n, E, batch, shard count): each kind meets every PRF, from its smallest table up to n = 2^14; batches
# around the lane split (< 32), the XOR key quads (1 to 3 keys padded), the leaf cache's 17 keys and its chunks
# (leaf_cache_mb = 1), entry sizes around the 16 / 32 / 64-column passes
SHAPES = {
    "standard": [(D, 2, 1, 1, 1), (S, 64, 16, 3, 2), (C, 1 << 10, 20, 5, 8), (A, 1 << 12, 33, 17, 1),
                 (D, 1 << 14, 128, 33, 2), (S, 1 << 13, 128, 100, 1), (C, 1 << 14, 16, 100, 8), (A, 1 << 14, 128, 17, 2)],
    "et": [(S, 8, 16, 1, 1), (C, 32, 1, 3, 2), (A, 1 << 10, 20, 5, 8), (D, 1 << 12, 33, 17, 1),
           (S, 1 << 14, 128, 33, 2), (C, 1 << 13, 128, 100, 1), (A, 1 << 14, 16, 100, 8), (D, 1 << 14, 128, 17, 2)],
    "xor": [(A, 256, 1, 1, 1), (D, 512, 16, 3, 2), (S, 1 << 12, 20, 5, 8), (C, 1 << 12, 33, 17, 1),
            (A, 1 << 14, 128, 33, 2), (D, 1 << 13, 128, 100, 1), (S, 1 << 14, 16, 100, 8), (C, 1 << 14, 20, 1, 2)],
}
PAIR_CASES = [(k, s) for k in PM.KINDS for s in SHAPES[k]]


@pytest.mark.parametrize("kind,shape", PAIR_CASES, ids=[shape_id(k, s) for k, s in PAIR_CASES])
def test_option_pairs(kind, shape):
    prf, n, e, batch, g = shape
    table = random_table(n, e, seed=n + e + batch)
    alphas = alphas_for(n, batch, seed=batch + g)
    a, b = PM.gen_keys(kind, n, alphas, prf, seed=n + batch)
    whole = PM.expected(kind, prf, a, table)
    assert np.array_equal(PM.reconstruct(kind, whole, PM.expected(kind, prf, b, table)), table[alphas])
    shares = PM.expected_shares(kind, prf, a) if g == 1 else None
    rows = PM.pairwise_rows(0)
    parts = [[] for _ in rows]
    for r in range(g):
        want = whole if g == 1 else PM.expected(kind, prf, a, table, r, g)
        ctx = context(kind, table, r, g)
        for i, row in enumerate(rows):       # one live context: every plan follows another
            set_options(ctx, row)
            entry = ENTRIES[i % len(ENTRIES)]
            where = "%s shard %d/%d, row %d %s, %s" % (shape_id(kind, shape), r, g, i, row, entry)
            got = evaluate(ctx, kind, entry, a, prf)
            assert np.array_equal(got, want), where
            parts[i].append(got)
            if g == 1:
                assert np.array_equal(expand(ctx, kind, a, prf), shares), where + ", expand_device"
        ctx.close()
    for i, row in enumerate(rows):
        assert np.array_equal(PM.combine(kind, parts[i]), whole), "%s row %d %s: shards" % (shape_id(kind, shape), i, row)


TOP_ROWS = [{"top_log2": t, "balance_top": bt, "one_launch": ol, "frontier_mb": mb}
            for t in range(8) for bt in (0, 1) for ol in (1, 0) for mb in (1, 256)]
PRF_CASES = [(k, p) for k in PM.KINDS for p in (D, S, C, A)]


def prf_id(kind, prf):
    return "%s-%s" % (kind, B.PRF_NAMES[prf])


@pytest.mark.parametrize("kind,prf", PRF_CASES, ids=[prf_id(k, p) for k, p in PRF_CASES])
def test_tree_top(kind, prf):
    """n = 2^16: 1, 40 and 9000 keys (282 key groups of 32: more than the blocks of any PRF's grid, so the
    one-launch kernel takes the host's per-block quota of tree-top items); n = 2^20 on a sparse table, whole
    and in 4 shards"""
    n, e = 1 << 16, 16
    table = random_table(n, e, seed=16 + prf)
    alphas = alphas_for(n, 9000, seed=prf)
    a, b = PM.gen_keys(kind, n, alphas, prf, seed=prf)
    last = len(a) - 32
    sample = np.random.RandomState(prf).choice(np.arange(40, last), size=180, replace=False)
    check = np.unique(np.concatenate([np.arange(40), np.arange(last, len(a)), sample]))
    want = PM.expected(kind, prf, a[check], table)
    ctx = context(kind, table)
    b_res = None
    for i, row in enumerate(TOP_ROWS):
        set_options(ctx, row)
        where = "%s n=2^16 row %d %s" % (prf_id(kind, prf), i, row)
        for batch in (1, 40):
            assert np.array_equal(ctx.eval(a[:batch], prf), want[:batch]), "%s, %d keys" % (where, batch)
        got = ctx.eval(a, prf)             # the first, in one launch, grows the tree-top tickets past 64
        assert np.array_equal(got[check], want), where + ", 9000 keys"
        if b_res is None:
            b_res = ctx.eval(b, prf)
        bad = np.nonzero((PM.reconstruct(kind, got, b_res) != table[alphas]).any(axis=1))[0]
        assert len(bad) == 0, "%s, 9000 keys: keys %s do not reconstruct" % (where, bad[:8].tolist())
    ctx.close()

    n, g = 1 << 20, 4
    alphas = alphas_for(n, 40, seed=20 + prf)
    sp = PM.Sparse(kind, n, e, alphas, shard_counts=(g,), seed=prf)
    table = sp.table()
    a, _ = PM.gen_keys(kind, n, alphas, prf, seed=20 + prf)
    whole = PM.expected(kind, prf, a, sp)
    for count in (1, g):
        parts = [[] for _ in TOP_ROWS]
        for r in range(count):
            want = whole if count == 1 else PM.expected(kind, prf, a, sp, r, count)
            ctx = context(kind, table, r, count)
            for i, row in enumerate(TOP_ROWS):
                set_options(ctx, row)
                got = ctx.eval(a, prf)
                assert np.array_equal(got, want), "%s n=2^20 sparse shard %d/%d row %d %s" % (prf_id(kind, prf), r, count, i, row)
                parts[i].append(got)
            ctx.close()
        for i, row in enumerate(TOP_ROWS):
            assert np.array_equal(PM.combine(kind, parts[i]), whole), "%s n=2^20 %d shards row %d %s" % (prf_id(kind, prf), count, i, row)


ITEM_CASES = [(k, p) for k in PM.KINDS for p in (A, C)]


@pytest.mark.parametrize("kind,prf", ITEM_CASES, ids=[prf_id(k, p) for k, p in ITEM_CASES])
def test_work_item_sizes(kind, prf):
    """subtree_log2 1..16 (clamped to the depth and to the deepest stack the layout holds), with and without
    the frontier, for lane-split batches of 2 and 3 keys and for 40 keys.  Standard AES keys take the broadcast
    kernel only with 1 or 2 keys per warp; 3 and 40 keys take the column-split kernel, whose stack is split
    around the T-tables at other levels."""
    e = 16
    for n in (1 << 16, 1 << 20) + ((1 << 24,) if prf == A else ()):
        alphas = alphas_for(n, 40, seed=n % 1000 + prf)
        if n == 1 << 16:
            table = random_table(n, e, seed=prf)
            ref = table
        else:
            ref = PM.Sparse(kind, n, e, alphas, seed=prf)
            table = ref.table()
        a, b = PM.gen_keys(kind, n, alphas, prf, seed=prf)
        want = PM.expected(kind, prf, a, ref)
        ctx = context(kind, table)
        del table
        assert np.array_equal(PM.reconstruct(kind, want, ctx.eval(b, prf)), ref[alphas])
        for s in range(1, 17):
            for frontier in (0, 1):
                ctx.set_option("subtree_log2", s)
                ctx.set_option("frontier", frontier)
                for batch in (2, 3, 40):
                    assert np.array_equal(ctx.eval(a[:batch], prf), want[:batch]), \
                        "%s n=2^%d subtree_log2=%d frontier=%d, %d keys" % (prf_id(kind, prf), n.bit_length() - 1, s, frontier, batch)
        ctx.close()


def _acc(kind, base, res):
    b, r = base.view(np.uint32), res.view(np.uint32)
    return (b ^ r if kind == "xor" else b + r).view(np.int32)


@pytest.mark.parametrize("kind", PM.KINDS)
def test_accumulate(kind):
    """(a) eval_device_acc adds (XOR-shared: XORs) into a non-zero buffer, in one launch or several, for a
    lane-split batch and for a wide one (standard and early-terminated: leaf-cache chunks of 64 keys and an
    uncached 16-key tail, MAC passes staged by cp.async.bulk or by registers); (b) the shard contexts of one
    table add their partials into one zeroed buffer on one stream, which ends as the whole table's result"""
    n = 1 << 12
    rng = np.random.RandomState(3)
    for prf, e, batch, opts in ((D, 20, 3, {}), (A, 128, 80, {"leaf_cache_mb": 1})):
        table = random_table(n, e, seed=e)
        alphas = alphas_for(n, batch, seed=e)
        a, _ = PM.gen_keys(kind, n, alphas, prf, seed=e)
        want = PM.expected(kind, prf, a, table)
        keys_dev = torch.from_numpy(a).cuda()
        base = rng.randint(-2**31, 2**31, size=(batch, e), dtype=np.int64).astype(np.int32)
        ctx = context(kind, table)
        set_options(ctx, opts)
        for one_launch in (0, 1):
            for mac_tma in (0, 1):
                ctx.set_option("one_launch", one_launch)
                ctx.set_option("mac_tma", mac_tma)
                out = torch.from_numpy(base).cuda()
                torch.cuda.synchronize()
                ctx.eval_device(keys_dev.data_ptr(), batch, prf, out.data_ptr(), accumulate=True)
                torch.cuda.synchronize()
                assert np.array_equal(out.cpu().numpy(), _acc(kind, base, want)), \
                    "%s E=%d %d keys one_launch=%d mac_tma=%d" % (kind, e, batch, one_launch, mac_tma)
        ctx.close()

    e, batch, prf = 40, 80, C
    table = random_table(n, e, seed=7)
    alphas = alphas_for(n, batch, seed=7)
    a, _ = PM.gen_keys(kind, n, alphas, prf, seed=7)
    whole = PM.expected(kind, prf, a, table)
    keys_dev = torch.from_numpy(a).cuda()
    for g in (2, 8):
        ctxs = [context(kind, table, r, g) for r in range(g)]
        for r, ctx in enumerate(ctxs):
            ctx.set_option("one_launch", r & 1)
        stream = torch.cuda.Stream()
        out = torch.zeros((batch, e), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        for ctx in ctxs:
            ctx.eval_device(keys_dev.data_ptr(), batch, prf, out.data_ptr(), stream=stream.cuda_stream, accumulate=True)
        stream.synchronize()
        assert np.array_equal(out.cpu().numpy(), whole), "%s: %d shards accumulated" % (kind, g)
        for ctx in ctxs:
            ctx.close()
