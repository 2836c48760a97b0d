"""Evaluation above n = 2^24, up to the documented n = 2^31, checked bit-exactly for every key.

Past 4 GiB of table the byte offsets of rows, leaf cache and shares no longer fit in 32 bits; at depth
26-31 leaf positions approach 2^31; the frontier cap and the leaf-cache cap start to bind.  Dense
oracles cost O(n) per key there, so the tables are sparse (tests/sparse_oracle.py): zero except on a
support chosen in position space (a row in every 1/4096 of the device table, the rows around every
4 GiB and shard boundary, each key's target and its neighbours in the tree), and the exact result is
a sum over the support of per-index oracle walks.  One dense leg at n = 2^28 compares the fused result
with the expanded shares over the whole domain.

Each test checks that the free device memory covers its contexts and skips, naming the size, when
it does not; contexts are closed before the next one is made.
"""
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
import sparse_oracle as S  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu

GiB = 1 << 30
MARGIN = 2 * GiB
PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


def require(torch, nbytes, what):
    """skip unless the device has nbytes free beyond a margin"""
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + MARGIN:
        pytest.skip("%s needs %.1f GiB of device memory, %.1f GiB free" % (what, nbytes / GiB, free / GiB))


def padded_bytes(rows, e):
    """device table: rows padded to 16, 32 or a multiple of 64 int32"""
    pad = 16 if e <= 16 else 32 if e <= 32 else (e + 63) & ~63
    return rows * pad * 4


def create_bytes(rows, e):
    """a context's table plus the unpadded staging copy that creation holds briefly"""
    return padded_bytes(rows, e) + rows * e * 4


def keys(n, batch, prf, seed, et=False, special=()):
    """key pairs for random targets, the first ones at `special`"""
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=batch).astype(np.int64)
    special = list(special)[:batch]
    alphas[:len(special)] = special
    seeds = rng.randint(0, 256, size=44 * batch).astype(np.uint8).tobytes()
    a, b = (B.gen_batch_et if et else B.gen_batch_secure)(alphas, n, seeds, prf)
    return a, b, alphas


def specials(n, rows_per_leaf=1):
    """targets at the ends of the domain and at the first and last rows of the 4 GiB marks"""
    depth = (n // rows_per_leaf).bit_length() - 1
    out = [0, n - 1]
    for pos in (1 << 26) // rows_per_leaf, (1 << 30) // rows_per_leaf:
        for p in (pos - 1, pos):
            if p < n // rows_per_leaf:
                out.append(int(S.bitrev(p, depth)) * rows_per_leaf + rows_per_leaf - 1)
    return out


class Sparse:
    """a sparse table: support units, their rows and values, the host table, and the reference"""

    def __init__(self, orc, n, e, targets, rows_per_leaf=1, shard_counts=(), seed=0):
        self.orc, self.n, self.e, self.rpl = orc, n, e, rows_per_leaf
        self.depth = (n // rows_per_leaf).bit_length() - 1
        self.units = S.support(self.depth, np.asarray(targets) // rows_per_leaf, rows_per_leaf, shard_counts, seed)
        self.rows = S.rows_of(self.units, rows_per_leaf)
        self.vals = S.values(len(self.rows), e, seed + 1)
        self._host = None
        self._shares = {}

    @property
    def host(self):
        if self._host is None:
            self._host = S.host_table(self.n, self.rows, self.vals)
        return self._host

    def device(self, torch):
        t = torch.zeros((self.n, self.e), dtype=torch.int32, device="cuda")
        t[torch.from_numpy(self.rows).cuda()] = torch.from_numpy(self.vals).cuda()
        torch.cuda.synchronize()
        return t

    def update(self, idx, rows):
        """apply table[idx[j]] := rows[j] (idx in the support) to the reference values and host table"""
        where = {int(r): k for k, r in enumerate(self.rows)}
        for i, r in zip(idx, rows):
            self.vals[where[int(i)]] = r
            if self._host is not None:
                self._host[int(i)] = r

    def ref(self, keys, prf, shard=None):
        """the exact result of `keys` (of one shard), from per-index shares computed once per key set"""
        keys = np.ascontiguousarray(keys, np.int32).reshape(-1, B.KEY_WORDS)
        tag = (prf, hash(keys.tobytes()))
        if tag not in self._shares:
            self._shares[tag] = S.shares(self.orc, keys, prf, self.units, self.rpl)
        sh, vals = self._shares[tag], self.vals
        if shard is not None:
            keep = np.repeat(S.owned(self.units, shard[0], shard[1]), self.rpl)
            sh, vals = sh[:, keep], vals[keep]
        return S.dot_u32(sh, vals)

    def at(self, alphas):
        where = {int(r): k for k, r in enumerate(self.rows)}
        return self.vals[[where[int(a)] for a in alphas]]


def check(sp, ctx_eval, a, b, alphas, prf, shard=None):
    ra, rb = ctx_eval(a), ctx_eval(b)
    assert np.array_equal(ra, sp.ref(a, prf, shard)), "server A shares differ from the sparse reference"
    assert np.array_equal(rb, sp.ref(b, prf, shard)), "server B shares differ from the sparse reference"
    if shard is None:
        assert np.array_equal(S.sub_u32(ra, rb), sp.at(alphas))
    return ra, rb


def create_et_from_device(ptr, n, e, shard_rank=0, shard_count=1):
    ctx = B.Context.__new__(B.Context)
    ctx.n, ctx.entry_size = n, e
    ctx.handle = C.c_void_p()
    B._check(B.lib().b200dpf_create_et(C.byref(ctx.handle), C.c_void_p(ptr), n, e, 0, shard_rank, shard_count),
             "b200dpf_create_et")
    return ctx


# ---- n = 2^26, 16 columns: a 4 GiB table ---------------------------------------------------------------

def test_n26_e16_every_prf(oracle, torch_cuda):
    n, e = 1 << 26, 16
    require(torch_cuda, create_bytes(n, e), "n = 2^26, E = 16")
    sets = {}
    for prf in PRFS:
        for batch in (33, 3):
            sets[prf, batch] = keys(n, batch, prf, seed=100 + 10 * prf + batch, special=specials(n))
    sp = Sparse(oracle, n, e, np.concatenate([v[2] for v in sets.values()]), seed=1)
    ctx = B.Context(sp.host)
    try:
        for (prf, batch), (a, b, alphas) in sets.items():
            check(sp, lambda k: ctx.eval(k, prf), a, b, alphas, prf)
        # the knobs that change the traversal, and compact keys, on one PRF
        prf = B.PRF_CHACHA20
        a, b, alphas = sets[prf, 33]
        want = sp.ref(a, prf)
        for name, value, default in (("frontier", 0, 1), ("frontier_mb", 1, 256), ("one_launch", 0, 1)):
            ctx.set_option(name, value)
            assert np.array_equal(ctx.eval(a, prf), want), name
            assert np.array_equal(ctx.eval(a[:3], prf), want[:3]), name
            ctx.set_option(name, default)
        packed = b"".join(B.key_pack(k) for k in a)
        assert np.array_equal(ctx.eval_packed(packed, len(a), prf), want)
    finally:
        ctx.close()


# ---- n = 2^28, one column: a 16 GiB table ---------------------------------------------------------------

def _int64_dot_mod32(torch, shares, table):
    """shares int32 [B, n] x table int32 [n] -> int32 [B] mod 2^32, on the device in chunks"""
    out = torch.zeros(shares.shape[0], dtype=torch.int64, device="cuda")
    step = 1 << 25
    for c in range(0, shares.shape[1], step):
        prod = shares[:, c:c + step].to(torch.int64) * table[c:c + step].to(torch.int64)[None, :]
        out = (out + (prod & 0xFFFFFFFF).sum(dim=1)) & 0xFFFFFFFF
    return out.cpu().numpy().astype(np.uint32).view(np.int32)


@pytest.mark.parametrize("prf", (B.PRF_AES128, B.PRF_CHACHA20))
def test_n28_e1(oracle, torch_cuda, prf):
    torch = torch_cuda
    n, e = 1 << 28, 1
    require(torch, create_bytes(n, e) + 2 * n * 4 + n * 4, "n = 2^28, E = 1, with two expanded keys")
    a, b, alphas = keys(n, 64, prf, seed=200 + prf, special=specials(n))
    sp = Sparse(oracle, n, e, alphas, seed=2)
    ctx = B.Context(sp.host)
    try:
        check(sp, lambda k: ctx.eval(k, prf), a, b, alphas, prf)
        check(sp, lambda k: ctx.eval(k, prf), a[5:6], b[5:6], alphas[5:6], prf)
        # dense leg: two keys expanded over the whole domain
        kd = torch.from_numpy(np.stack([a[5], b[5]])).cuda()
        shares = torch.empty((2, n), dtype=torch.int32, device="cuda")
        ctx.expand_device(kd.data_ptr(), 2, prf, shares.data_ptr())
        torch.cuda.synchronize()
    finally:
        ctx.close()
    d = shares[0] - shares[1]
    nz = torch.nonzero(d).flatten().cpu().numpy()
    assert nz.tolist() == [int(alphas[5])] and int(d[int(alphas[5])]) == 1
    rows = torch.from_numpy(sp.rows).cuda()
    got = shares[:, rows].cpu().numpy()
    assert np.array_equal(got, oracle.eval_points(np.stack([a[5], b[5]]), prf, sp.rows))
    # the fused result on a dense random table against the expanded shares
    gen = torch.Generator(device="cuda").manual_seed(28 + prf)
    dense = torch.randint(-2**31, 2**31, (n, 1), dtype=torch.int32, device="cuda", generator=gen)
    ctx = B.Context.from_device_ptr(dense.data_ptr(), n, 1)
    try:
        fused = ctx.eval(np.stack([a[5], b[5]]), prf)
    finally:
        ctx.close()
    assert np.array_equal(fused[:, 0], _int64_dot_mod32(torch, shares, dense[:, 0]))
    assert S.sub_u32(fused[0], fused[1])[0] == dense[int(alphas[5]), 0].item()


# ---- wide entries: 40 columns at n = 2^26 (256-byte rows, a 16 GiB table) --------------------------------

def test_n26_wide_entries_leaf_cache(oracle, torch_cuda):
    """A key group's leaf cache (32 keys x n x 4 B = 8 GiB) under the default 16 GiB cap, over a
    4 GiB cap (one group alone overflows it: every 64-column slice re-expands), and both MAC kernels."""
    n, e, prf = 1 << 26, 40, B.PRF_CHACHA20
    cache = 2 * 32 * n * 4
    require(torch_cuda, max(create_bytes(n, e), padded_bytes(n, e) + cache), "n = 2^26, E = 40 with its leaf cache")
    a, b, alphas = keys(n, 33, prf, seed=300, special=specials(n))
    sp = Sparse(oracle, n, e, alphas, seed=3)
    want = sp.ref(a, prf)
    ctx = B.Context(sp.host)
    try:
        for opts in ({}, {"mac_tma": 0}, {"mac_tma": 1}, {"leaf_cache_mb": 4096}, {"leaf_cache": 0}):
            for k, v in opts.items():
                ctx.set_option(k, v)
            assert np.array_equal(ctx.eval(a, prf), want), opts
            for k in opts:
                ctx.set_option(k, {"mac_tma": 1, "leaf_cache_mb": 16384, "leaf_cache": 1}[k])
        assert np.array_equal(S.sub_u32(want, ctx.eval(b, prf)), sp.at(alphas))
    finally:
        ctx.close()


@pytest.mark.parametrize("prf", PRFS)
def test_one_key_group_over_the_leaf_cache_cap(oracle, torch_cuda, prf):
    """The same branch at a small size: 2 MiB per key group against a 1 MiB cap."""
    n, e = 1 << 14, 128
    table = random_table(n, e, seed=301)
    a, b, alphas = keys(n, 33, prf, seed=302)
    ctx = B.Context(table)
    try:
        ctx.set_option("leaf_cache_mb", 1)
        ra = ctx.eval(a, prf)
        assert np.array_equal(S.sub_u32(ra, ctx.eval(b, prf)), table[alphas])
        ctx.set_option("leaf_cache_mb", 16384)
        assert np.array_equal(ctx.eval(a, prf), ra)
    finally:
        ctx.close()
    pick = [0, 32]
    assert np.array_equal(ra[pick], S.dot_u32(oracle.eval_points(a[pick], prf, np.arange(n)), table))


# ---- n = 2^31 in four shards (32 GiB each), with row updates --------------------------------------------

def _shards_2e31(oracle, torch, prf, et):
    n, e, shards = 1 << 31, 1, 4
    rpl = 4 if et else 1
    local = n // shards
    require(torch, n * 4 + create_bytes(local, e), "a 2^31-row shard (with the whole table on the device)")
    a, b, alphas = keys(n, 33, prf, seed=400 + prf + 7 * et, et=et, special=specials(n, rpl))
    sp = Sparse(oracle, n, e, alphas, rows_per_leaf=rpl, shard_counts=(shards,), seed=4 + et)
    # updates at both ends and around the 4 GiB (2^26-row) marks, all in the support
    upd = sorted({0, n - 1, n - 2} | {int(r) for r in specials(n, rpl)} |
                 {int(S.bitrev(k * ((1 << 26) // rpl) + d, 31 - 2 * et)) * rpl + (k % rpl)
                  for k in range(1, n // (1 << 26)) for d in (-1, 0)})
    upd = np.array(upd, np.int64)
    new_rows = S.values(len(upd), e, seed=41 + et)
    half = len(upd) // 2
    dev_table = sp.device(torch)
    idx_dev = torch.from_numpy(upd[half:]).cuda()
    rows_dev = torch.from_numpy(new_rows[half:]).cuda()
    before = [np.zeros((len(a), e), np.uint32) for _ in range(2)]
    parts = []
    for r in range(shards):
        if r % 2 == 0:
            ctx = B.Context(sp.host, shard_rank=r, shard_count=shards, early_termination=et)
        elif et:
            ctx = create_et_from_device(dev_table.data_ptr(), n, e, r, shards)
        else:
            ctx = B.Context.from_device_ptr(dev_table.data_ptr(), n, e, shard_rank=r, shard_count=shards)
        try:
            ra, rb = check(sp, lambda k: ctx.eval(k, prf), a, b, alphas, prf, shard=(r, shards))
            before[0] += ra.view(np.uint32)
            before[1] += rb.view(np.uint32)
            ctx.update_rows(upd[:half], new_rows[:half])
            ctx.update_rows_device(idx_dev.data_ptr(), rows_dev.data_ptr(), len(upd) - half)
            torch.cuda.synchronize()
            parts.append((ctx.eval(a, prf), ctx.eval(b, prf)))
        finally:
            ctx.close()
    whole_a, whole_b = sp.ref(a, prf), sp.ref(b, prf)
    assert np.array_equal(before[0].view(np.int32), whole_a)
    assert np.array_equal(before[1].view(np.int32), whole_b)
    assert np.array_equal(S.sub_u32(whole_a, whole_b), sp.at(alphas))
    sp.update(upd, new_rows)
    after = [np.zeros((len(a), e), np.uint32) for _ in range(2)]
    for r, (ra, rb) in enumerate(parts):
        assert np.array_equal(ra, sp.ref(a, prf, (r, shards))), ("updated shard", r)
        assert np.array_equal(rb, sp.ref(b, prf, (r, shards))), ("updated shard", r)
        after[0] += ra.view(np.uint32)
        after[1] += rb.view(np.uint32)
    assert np.array_equal(S.sub_u32(after[0].view(np.int32), after[1].view(np.int32)), sp.at(alphas))


@pytest.mark.parametrize("prf", (B.PRF_AES128, B.PRF_SALSA20))
def test_n31_four_shards(oracle, torch_cuda, prf):
    _shards_2e31(oracle, torch_cuda, prf, et=False)


# ---- early-terminated keys ----------------------------------------------------------------------------

def test_et_n28_e16(oracle, torch_cuda):
    n, e = 1 << 28, 16
    require(torch_cuda, create_bytes(n, e), "an early-terminated context of n = 2^28, E = 16")
    sets = {prf: keys(n, 33, prf, seed=500 + prf, et=True, special=specials(n, 4))
            for prf in (B.PRF_AES128, B.PRF_SALSA20)}
    sp = Sparse(oracle, n, e, np.concatenate([v[2] for v in sets.values()]), rows_per_leaf=4, seed=5)
    ctx = B.Context(sp.host, early_termination=True)
    try:
        for prf, (a, b, alphas) in sets.items():
            check(sp, lambda k: ctx.eval(k, prf), a, b, alphas, prf)
    finally:
        ctx.close()


@pytest.mark.parametrize("prf", (B.PRF_AES128, B.PRF_SALSA20))
def test_et_n31_four_shards(oracle, torch_cuda, prf):
    _shards_2e31(oracle, torch_cuda, prf, et=True)


# ---- grouped context: bins that start past 4 GiB ------------------------------------------------------

def test_grouped_bins_past_4gib(oracle, torch_cuda):
    sizes, e, prf = [1 << 26, 1 << 10, 1 << 14, 2], 16, B.PRF_AES128
    require(torch_cuda, create_bytes(sum(sizes), e), "a grouped context of 2^26 + 2^14 + 2^10 + 2 rows")
    per_bin = [keys(nb, 9, prf, seed=600 + g, special=specials(nb) if g == 0 else ()) for g, nb in enumerate(sizes)]
    sp = Sparse(oracle, sizes[0], e, per_bin[0][2], seed=6)
    small = [random_table(nb, e, seed=601 + g) for g, nb in enumerate(sizes[1:])]
    ka = np.concatenate([k[0] for k in per_bin])
    kb = np.concatenate([k[1] for k in per_bin])
    bins = np.repeat(np.arange(len(sizes), dtype=np.int32), 9)
    order = np.random.RandomState(602).permutation(len(bins))      # a mixed list of (bin, key)
    ka, kb, bins = ka[order], kb[order], bins[order]

    def want(keys_):
        out = np.zeros((len(keys_), e), np.int32)
        for g in range(len(sizes)):
            sel = bins == g
            if g == 0:
                out[sel] = sp.ref(keys_[sel], prf)
            else:
                t = small[g - 1]
                out[sel] = S.dot_u32(oracle.eval_points(keys_[sel], prf, np.arange(sizes[g])), t)
        return out

    ctx = B.GroupContext([sp.host] + small)
    try:
        assert ctx.nbins == 4
        ra, rb = ctx.eval(ka, bins, prf), ctx.eval(kb, bins, prf)
        assert np.array_equal(ra, want(ka)) and np.array_equal(rb, want(kb))
        # rows in every bin, bin 0's at the start, the end and around its own 2^26 end
        ub = np.array([0, 0, 0, 1, 1, 2, 2, 3, 3], np.int32)
        ui = np.array([0, sizes[0] - 1, int(sp.rows[len(sp.rows) // 2]), 0, sizes[1] - 1, 5, sizes[2] - 1, 0, 1], np.int64)
        rows = S.values(len(ub), e, seed=603)
        ctx.update_rows(ub, ui, rows)
        sp.update(ui[ub == 0], rows[ub == 0])
        for g in range(1, 4):
            small[g - 1][ui[ub == g]] = rows[ub == g]
        ra, rb = ctx.eval(ka, bins, prf), ctx.eval(kb, bins, prf)
        assert np.array_equal(ra, want(ka)) and np.array_equal(rb, want(kb))
    finally:
        ctx.close()


# ---- GPU key generation at every depth ---------------------------------------------------------------

@pytest.mark.parametrize("prf", PRFS)
def test_gpu_keygen_every_depth(torch_cuda, prf):
    torch = torch_cuda
    rng = np.random.RandomState(700 + prf)
    for depth in range(1, 32):
        n = 1 << depth
        alphas = np.array([0, n - 1] + list(rng.randint(0, n, size=3)), np.int64)
        seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
        ha, hb = B.gen_batch_secure(alphas, n, seeds, prf)
        ga, gb = B.gen_batch_gpu(alphas, n, seeds, prf)
        assert np.array_equal(ga, ha) and np.array_equal(gb, hb), depth
        da = torch.zeros((len(alphas), B.KEY_WORDS), dtype=torch.int32, device="cuda")
        db = torch.zeros_like(da)
        B.gen_batch_gpu(alphas, n, seeds, prf, out_ptrs=(da.data_ptr(), db.data_ptr()))
        torch.cuda.synchronize()
        assert np.array_equal(da.cpu().numpy(), ha) and np.array_equal(db.cpu().numpy(), hb), depth
