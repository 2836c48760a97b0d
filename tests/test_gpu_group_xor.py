"""Grouped (batch-PIR) evaluation of XOR-shared keys on the GPU (b200dpf_group_create_xor): shuffled lists
of (bin, key) pairs over bins of 256 to 2^14 rows, launches with many more work units than blocks and with
fewer, and a bin of 2^26 rows whose successors start past 4 GiB.  Every pair reconstructs its row
(a ^ b = table[bin][alpha]) and is checked against an ordinary XOR-shared context on its bin (bit for bit)
or the host evaluation, and some pairs of every bin against the per-index oracle (tests/xor_oracle.py)."""
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
import oracle  # noqa: E402
import sparse_oracle as S  # noqa: E402
import xor_oracle  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
SIZES = [256, 512, 1 << 10, 1 << 12, 1 << 14]
PER_BIN = [1, 3, 5, 33, 70]                  # partial key quads, and more than one 32-key group in two bins
ORACLE_PAIRS = 2
GiB = 1 << 30


@pytest.fixture(scope="module")
def orc():
    return oracle.Oracle()


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


def gen_pairs(sizes, per_bin, prf, seed):
    """shuffled (bin, key) pairs: key pairs of every bin (its first and last row among the targets)"""
    rng = np.random.RandomState(seed)
    ka, kb, bins, alphas = [], [], [], []
    for g, (n, cnt) in enumerate(zip(sizes, per_bin)):
        al = rng.randint(0, n, size=cnt).astype(np.int64)
        al[:2] = [0, n - 1][:cnt]
        a, b = B.gen_batch_xor(al, n, rng.randint(0, 256, size=44 * cnt).astype(np.uint8).tobytes(), prf)
        ka.append(a); kb.append(b); bins += [g] * cnt; alphas.append(al)
    order = rng.permutation(len(bins))
    return (np.concatenate(ka)[order], np.concatenate(kb)[order], np.array(bins, np.int32)[order],
            np.concatenate(alphas)[order])


def xor(a, b):
    return (a.view(np.uint32) ^ b.view(np.uint32)).view(np.int32)


def selected_rows(tables, bins, alphas):
    return np.stack([tables[g][a] for g, a in zip(bins, alphas)])


def host_result(keys, prf, table):
    """the host evaluation: XOR of the rows whose share bit is set"""
    return xor_oracle.xor_rows(np.stack([xor_oracle.unpack_bits(B.eval_cpu_xor(k, prf)) for k in keys]), table)


def check_against_bins(got, keys, bins, ctxs, prf):
    """every pair equals an ordinary XOR-shared context on its bin, bit for bit"""
    for g, ctx in enumerate(ctxs):
        sel = np.nonzero(bins == g)[0]
        assert np.array_equal(got[sel], ctx.eval(keys[sel], prf)), "bin %d" % g


_oracle_results = {}


def check_oracle(orc, got, keys, bins, tables, prf):
    for g, t in enumerate(tables):
        sel = np.nonzero(bins == g)[0][:ORACLE_PAIRS]
        assert len(sel) > 0
        tag = (prf, keys[sel].tobytes(), t.tobytes())
        if tag not in _oracle_results:
            _oracle_results[tag] = xor_oracle.eval_xor(orc, keys[sel], prf, t)
        assert np.array_equal(got[sel], _oracle_results[tag]), "bin %d" % g


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("e", [1, 5, 16, 33, 40])
def test_mixed_bins_bit_exact(orc, torch_cuda, prf, e):
    ka, kb, bins, alphas = gen_pairs(SIZES, PER_BIN, prf, seed=100 + prf)
    tables = [random_table(n, e, seed=10 * g + e) for g, n in enumerate(SIZES)]
    ctx = B.GroupContext(tables, xor=True)
    ctxs = [B.Context(t, xor=True) for t in tables]
    try:
        assert ctx.nbins == len(SIZES) and ctx.rows_per_leaf == 128
        ra = ctx.eval(ka, bins, prf)
        assert ctx.last_launches == (e + 15) // 16
        rb = ctx.eval(kb, bins, prf)
        assert np.array_equal(xor(ra, rb), selected_rows(tables, bins, alphas))
        check_against_bins(ra, ka, bins, ctxs, prf)
        check_against_bins(rb, kb, bins, ctxs, prf)
        check_oracle(orc, ra, ka, bins, tables, prf)
    finally:
        ctx.close()
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("prf", [B.PRF_CHACHA20, B.PRF_AES128])
def test_work_item_size_single_pair_single_group(torch_cuda, prf):
    ka, _, bins, _ = gen_pairs(SIZES, PER_BIN, prf, seed=200 + prf)
    tables = [random_table(n, 16, seed=300 + g) for g, n in enumerate(SIZES)]
    ctx = B.GroupContext(tables, xor=True)
    try:
        want = ctx.eval(ka, bins, prf)
        for s in (1, 2, 3, 7):                    # the work-item size is a tuning knob only
            ctx.set_subtree_log2(s)
            assert np.array_equal(ctx.eval(ka, bins, prf), want), s
        ctx.set_subtree_log2(0)
        for j in range(3):                        # a single pair
            assert np.array_equal(ctx.eval(ka[j:j + 1], bins[j:j + 1], prf), want[j:j + 1])
        for g in (2, 3):                          # a single key group: 5 keys, then 32 of 33
            sel = np.nonzero(bins == g)[0][:32]
            assert np.array_equal(ctx.eval(ka[sel], bins[sel], prf), want[sel]), g
    finally:
        ctx.close()


@pytest.mark.parametrize("sizes,per_bin", [
    ([256] * 1024, [2] * 1024),                   # 1,024 one-item key groups: many more units than blocks
    ([1 << 12, 1 << 10], [3, 2]),                 # two key groups of 16 and 4 items: fewer units than blocks
])
def test_unit_counts(torch_cuda, sizes, per_bin):
    prf, e = B.PRF_AES128, 16
    ka, kb, bins, alphas = gen_pairs(sizes, per_bin, prf, seed=len(sizes))
    tables = [random_table(n, e, seed=800 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, xor=True)
    try:
        ra, rb = ctx.eval(ka, bins, prf), ctx.eval(kb, bins, prf)
        assert np.array_equal(xor(ra, rb), selected_rows(tables, bins, alphas))
        for g in range(0, len(sizes), max(1, len(sizes) // 16)):
            sel = np.nonzero(bins == g)[0]
            assert np.array_equal(ra[sel], host_result(ka[sel], prf, tables[g])), g
    finally:
        ctx.close()


def test_refusals(torch_cuda):
    prf = B.PRF_AES128
    sizes = [256, 1 << 10]
    tables = [random_table(n, 16, seed=400 + g) for g, n in enumerate(sizes)]
    ka, _, bins, _ = gen_pairs(sizes, [6, 6], prf, seed=401)
    std_a, _ = B.gen_batch_secure(np.array([3], np.int64), 256, bytes(range(44)), prf)
    et_a, _ = B.gen_batch_et(np.array([3], np.int64), 256, bytes(range(44)), prf)
    ctx = B.GroupContext(tables, xor=True)
    try:
        want = ctx.eval(ka, bins, prf)
        one = np.concatenate([bins, [0]]).astype(np.int32)
        with pytest.raises(B.B200DPFError, match=r"\(-1\).*key 12 is a standard key; this XOR-shared context takes keys "
                                                 r"of b200dpf_gen_xor"):
            ctx.eval(np.concatenate([ka, std_a]), one, prf)
        with pytest.raises(B.B200DPFError, match=r"\(-1\).*key 12 is an early-terminated key; this XOR-shared context"):
            ctx.eval(np.concatenate([ka, et_a]), one, prf)
        with pytest.raises(B.B200DPFError, match=r"\(-1\).*not an XOR-shared key for n=1024 \(its n: 256\)"):
            ctx.eval(ka, np.where(bins == 0, 1, bins).astype(np.int32), prf)   # a 256-row key on the 1024-row bin
        with pytest.raises(B.B200DPFError, match=r"\(-1\).*bin 2 out of range"):
            ctx.eval(ka, np.full(len(ka), 2, np.int32), prf)
        with pytest.raises(B.B200DPFError, match=r"\(-4\).*grouped context"):
            B.Context.eval(ctx, ka[:1], prf)
        assert np.array_equal(ctx.eval(ka, bins, prf), want)   # nothing above disturbed the context
    finally:
        ctx.close()
    std = B.GroupContext(tables)                  # the other grouped contexts still refuse XOR-shared keys
    et = B.GroupContext(tables, early_termination=True)
    try:
        with pytest.raises(B.B200DPFError, match=r"\(-1\).*generated for n=-1.*it is an XOR-shared key"):
            std.eval(ka, bins, prf)
        with pytest.raises(B.B200DPFError, match=r"\(-1\).*is an XOR-shared key; this early-terminated context"):
            et.eval(ka, bins, prf)
    finally:
        std.close()
        et.close()


@pytest.mark.parametrize("prf", [B.PRF_SALSA20, B.PRF_AES128])
def test_group_update_rows(orc, torch_cuda, prf):
    e = 5
    ka, kb, bins, alphas = gen_pairs(SIZES, PER_BIN, prf, seed=500 + prf)
    tables = [random_table(n, e, seed=510 + g) for g, n in enumerate(SIZES)]
    ctx = B.GroupContext(tables, xor=True)
    try:
        before = ctx.eval(ka, bins, prf)
        ub, ui = [], []
        for g, n in enumerate(SIZES):             # the first and last row of every bin, one in between
            ub += [g, g, g]
            ui += [0, n - 1, (n // 2) | 1]
        ub += [3] * 4                             # both sides of a 128-row leaf boundary of bin 3
        ui += [127, 128, 1023, 1024]
        ub += [4, 2, 4]                           # a repeated index of bin 4: the last occurrence wins
        ui += [1000, 9, 1000]
        ub, ui = np.array(ub, np.int32), np.array(ui, np.int64)
        rows = random_table(len(ub), e, seed=520)
        bad = [(np.append(ub, len(SIZES)).astype(np.int32), np.append(ui, 0)),     # bin out of range
               (np.append(ub, 2).astype(np.int32), np.append(ui, SIZES[2])),       # index past the bin
               (np.append(ub, 1).astype(np.int32), np.append(ui, -1))]
        for bb, bi in bad:
            with pytest.raises(B.B200DPFError, match=r"\(-1\)"):
                ctx.update_rows(bb, bi, np.concatenate([rows, rows[:1]]))
            assert np.array_equal(ctx.eval(ka, bins, prf), before)   # nothing was applied
        ctx.update_rows(ub, ui, rows)
        for g, i, r in zip(ub, ui, rows):         # in order: the last occurrence wins
            tables[g][i] = r
        ra, rb = ctx.eval(ka, bins, prf), ctx.eval(kb, bins, prf)
        assert not np.array_equal(ra, before)
        assert np.array_equal(xor(ra, rb), selected_rows(tables, bins, alphas))
        check_oracle(orc, ra, ka, bins, tables, prf)
        for g, t in enumerate(tables):            # every pair against the host evaluation
            sel = np.nonzero(bins == g)[0]
            assert np.array_equal(ra[sel], host_result(ka[sel], prf, t)), g
    finally:
        ctx.close()


def test_bins_past_4_gib(orc, torch_cuda):
    """a 2^26-row first bin (4 GiB of 64-byte rows): the small bins' rows start past 4 GiB.  The big bin is
    zero except on a support set (its alphas, both sides of leaf boundaries, the rows the device table holds
    last), so its expected result is the XOR of the support rows whose share bit is set."""
    torch = torch_cuda
    prf, e = B.PRF_AES128, 16
    sizes = [1 << 26, 256, 1 << 10, 1 << 14]
    need = sum(sizes) * 64 + (1 << 26) * e * 4
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    if free < need + 2 * GiB:
        pytest.skip("needs %.1f GiB of device memory, %.1f GiB free" % (need / GiB, free / GiB))
    ka, kb, bins, alphas = gen_pairs(sizes, [5, 6, 7, 6], prf, seed=600)
    n0, depth0 = sizes[0], 26 - 7

    def natural(dev_row):
        leaf = int(format(dev_row >> 7, "0%db" % depth0)[::-1], 2)
        return (leaf << 7) | (dev_row & 127)

    support = set(int(a) for a in alphas[bins == 0]) | {natural(r) for r in (n0 - 2, n0 - 1)}
    for c in (128, 1 << 12, 1 << 20, n0 // 2 + (1 << 24)):
        support.update((c - 1, c))
    support = np.array(sorted(s for s in support if 0 <= s < n0), np.int64)
    vals0 = S.values(len(support), e, seed=7)
    big = S.host_table(n0, support, vals0)
    small = [random_table(n, e, seed=610 + g) for g, n in enumerate(sizes[1:])]

    def want(keys):
        out = np.zeros((len(keys), e), np.int32)
        sel = np.nonzero(bins == 0)[0]
        bits = np.stack([xor_oracle.unpack_bits(B.eval_cpu_xor(k, prf))[support] for k in keys[sel]])
        out[sel] = xor_oracle.xor_rows(bits, vals0)
        for g, t in enumerate(small, 1):
            sel = bins == g
            out[sel] = host_result(keys[sel], prf, t)
        return out

    ctx = B.GroupContext([big] + small, xor=True)
    del big
    try:
        ra, rb = ctx.eval(ka, bins, prf), ctx.eval(kb, bins, prf)
        assert np.array_equal(ra, want(ka)) and np.array_equal(rb, want(kb))
        k0 = np.nonzero(bins == 0)[0][0]          # spot checks of the host bits against the per-index oracle
        bits = xor_oracle.unpack_bits(B.eval_cpu_xor(ka[k0], prf))
        for i in support[::3]:
            assert int(bits[i]) == xor_oracle.share_bit(orc, ka[k0], int(i), prf)
        # rows of every bin: bin 0's last device row and a leaf boundary, the ends of the others
        ub = np.array([0, 0, 0, 1, 1, 2, 2, 3, 3], np.int32)
        ui = np.array([natural(n0 - 1), 127, 128, 0, sizes[1] - 1, 0, sizes[2] - 1, 5, sizes[3] - 1], np.int64)
        assert set(ui[:3].tolist()) <= set(support.tolist())
        rows = S.values(len(ub), e, seed=8)
        ctx.update_rows(ub, ui, rows)
        where = {int(r): k for k, r in enumerate(support)}
        for g, i, r in zip(ub, ui, rows):
            if g == 0:
                vals0[where[int(i)]] = r
            else:
                small[g - 1][i] = r
        ra, rb = ctx.eval(ka, bins, prf), ctx.eval(kb, bins, prf)
        assert np.array_equal(ra, want(ka)) and np.array_equal(rb, want(kb))
        sel = bins != 0
        assert np.array_equal(xor(ra, rb)[sel], np.stack([small[g - 1][a] for g, a in zip(bins[sel], alphas[sel])]))
    finally:
        ctx.close()


def test_dpf_cpp_path(torch_cuda):
    torch = torch_cuda
    import dpf
    cpp = dpf.dpf_cpp
    prf = B.PRF_CHACHA20
    sizes = [256, 1 << 10, 1 << 12]
    tables = [random_table(n, 16, seed=700 + g) for g, n in enumerate(sizes)]
    ka, kb, bins, alphas = gen_pairs(sizes, [5, 5, 5], prf, seed=701)
    buf = cpp.group_init_xor([torch.from_numpy(t) for t in tables], 0)
    try:
        assert cpp.rows_per_leaf(buf) == 128
        ra = cpp.group_eval(torch.from_numpy(ka), torch.from_numpy(bins), buf, prf).numpy()
        rb = cpp.group_eval(torch.from_numpy(kb), torch.from_numpy(bins), buf, prf).numpy()
        assert np.array_equal(xor(ra, rb), selected_rows(tables, bins, alphas))
        row = random_table(1, 16, seed=702)
        g, a = int(bins[0]), int(alphas[0])
        cpp.group_update_rows(torch.tensor([g], dtype=torch.int32), torch.tensor([a], dtype=torch.int64),
                              torch.from_numpy(row), buf)
        tables[g][a] = row[0]
        ra = cpp.group_eval(torch.from_numpy(ka), torch.from_numpy(bins), buf, prf).numpy()
        rb = cpp.group_eval(torch.from_numpy(kb), torch.from_numpy(bins), buf, prf).numpy()
        assert np.array_equal(xor(ra, rb), selected_rows(tables, bins, alphas))
    finally:
        cpp.eval_free(buf)
