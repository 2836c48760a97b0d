"""Device-resident grouped (batch-PIR) evaluation on the GPU (b200dpf_group_eval_device): keys and results in
device memory, enqueued on a stream with no host synchronisation, for all three kinds of key.  Every result is
compared bit for bit with b200dpf_group_eval on the same keys and bins, and every pair reconstructs its row
(a - b, or a ^ b, = table[bin][alpha]).  Also covered: the work-item size knob, single pairs and key groups,
many and few work units, back-to-back calls on one and two streams mixed with host evaluations and row
updates, a call that returns while its stream is still busy, a bin whose successors start past 4 GiB, and
the three Python surfaces with their refusals."""
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
import sparse_oracle as S  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
PER_BIN = [1, 3, 5, 33, 70]                  # partial key groups, and more than one 32-key group in two bins
GiB = 1 << 30

# per kind: GroupContext keyword, bin sizes of the mixed-bin tests (the smallest each kind takes), key generator
KINDS = {
    "standard": ({}, [2, 64, 1 << 10, 1 << 12, 1 << 14]),
    "et": ({"early_termination": True}, [8, 64, 1 << 10, 1 << 12, 1 << 14]),
    "xor": ({"xor": True}, [256, 512, 1 << 10, 1 << 12, 1 << 14]),
}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


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


def reconstruct(kind, a, b):
    if kind == "xor":
        return (a.view(np.uint32) ^ b.view(np.uint32)).view(np.int32)
    return (a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32)


def selected_rows(tables, bins, alphas):
    return np.stack([tables[g][a] for g, a in zip(bins, alphas)])


def device_eval(torch, ctx, keys, bins, prf, stream=None):
    """GroupContext.eval_device on keys uploaded with torch; the result back on the host"""
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys)).cuda()
    out = torch.full((len(keys), ctx.entry_size), -1, dtype=torch.int32, device="cuda")
    st = stream if stream is not None else torch.cuda.current_stream()
    ctx.eval_device(keys_dev.data_ptr(), bins, prf, out.data_ptr(), st.cuda_stream)
    st.synchronize()
    return out.cpu().numpy()


def check_pairs(torch, kind, ctx, tables, ka, kb, bins, alphas, prf):
    """both sides bit-exact against the host path, and the pairs reconstruct their rows"""
    ra, rb = device_eval(torch, ctx, ka, bins, prf), device_eval(torch, ctx, kb, bins, prf)
    assert ctx.last_launches == (ctx.entry_size + 15) // 16      # the evaluation launches, timed alone
    assert ctx.last_device_ms > 0
    assert np.array_equal(ra, ctx.eval(ka, bins, prf))
    assert np.array_equal(rb, ctx.eval(kb, bins, prf))
    assert np.array_equal(reconstruct(kind, ra, rb), selected_rows(tables, bins, alphas))
    return ra


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("e", [1, 5, 16, 33, 40])
@pytest.mark.parametrize("kind", list(KINDS))
def test_mixed_bins_bit_exact(torch_cuda, kind, e, prf):
    kw, sizes = KINDS[kind]
    ka, kb, bins, alphas = gen_pairs(kind, sizes, PER_BIN, prf, seed=100 + prf)
    tables = [random_table(n, e, seed=10 * g + e) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **kw)
    try:
        check_pairs(torch_cuda, kind, ctx, tables, ka, kb, bins, alphas, prf)
    finally:
        ctx.close()


@pytest.mark.parametrize("prf", [B.PRF_CHACHA20, B.PRF_AES128])
@pytest.mark.parametrize("kind", ["standard", "et"])
def test_wide_entries(torch_cuda, kind, prf):
    kw, sizes = KINDS[kind]
    ka, kb, bins, alphas = gen_pairs(kind, sizes, PER_BIN, prf, seed=150 + prf)
    tables = [random_table(n, 200, seed=160 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **kw)
    try:
        check_pairs(torch_cuda, kind, ctx, tables, ka, kb, bins, alphas, prf)
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_work_item_size_single_pair_single_group(torch_cuda, kind):
    prf = B.PRF_AES128 if kind == "xor" else B.PRF_CHACHA20
    kw, sizes = KINDS[kind]
    ka, _, bins, _ = gen_pairs(kind, sizes, PER_BIN, prf, seed=200 + prf)
    tables = [random_table(n, 16, seed=300 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **kw)
    try:
        want = ctx.eval(ka, bins, prf)
        for s in (1, 2, 3, 7):                    # the work-item size is a tuning knob only
            ctx.set_subtree_log2(s)
            assert np.array_equal(device_eval(torch_cuda, ctx, ka, bins, prf), want), s
        ctx.set_subtree_log2(0)
        for j in range(3):                        # a single pair
            assert np.array_equal(device_eval(torch_cuda, ctx, ka[j:j + 1], bins[j:j + 1], prf), want[j:j + 1])
        for g in (2, 3):                          # a single key group: 5 keys, then 32 of 33
            sel = np.nonzero(bins == g)[0][:32]
            assert np.array_equal(device_eval(torch_cuda, ctx, ka[sel], bins[sel], prf), want[sel]), g
    finally:
        ctx.close()


@pytest.mark.parametrize("sizes,per_bin", [
    ([256] * 1024, [2] * 1024),                   # 1,024 one-item key groups: many more units than blocks
    ([1 << 12, 1 << 10], [3, 2]),                 # two key groups of 16 and 4 items: fewer units than blocks
])
def test_xor_unit_counts(torch_cuda, sizes, per_bin):
    prf, e = B.PRF_AES128, 16
    ka, kb, bins, alphas = gen_pairs("xor", sizes, per_bin, prf, seed=len(sizes))
    tables = [random_table(n, e, seed=800 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, xor=True)
    try:
        check_pairs(torch_cuda, "xor", ctx, tables, ka, kb, bins, alphas, prf)
    finally:
        ctx.close()


@pytest.mark.parametrize("nstreams", [1, 2])
@pytest.mark.parametrize("kind", list(KINDS))
def test_back_to_back_without_syncs(torch_cuda, kind, nstreams):
    """ten device calls with no synchronisation in between, of varying bin mixes and sizes (nkeys grows past
    every staging and scratch buffer's first size mid-sequence), with a host evaluation and a row update
    among them; one synchronisation at the end, then every result against its expected value"""
    torch = torch_cuda
    prf, e = B.PRF_AES128, 20
    kw, sizes = KINDS[kind]
    sizes = sizes[1:]                             # 4 bins
    tables = [random_table(n, e, seed=900 + g) for g, n in enumerate(sizes)]
    rng = np.random.RandomState(901 + nstreams)
    counts = [5, 40, 200, 37, 1500, 3, 700, 2600, 64, 1200]
    batches = []
    for i, cnt in enumerate(counts):
        nb = 1 + i % len(sizes)                   # the bins this batch touches
        bins = rng.randint(0, nb, size=cnt).astype(np.int32)
        alphas = np.array([rng.randint(0, sizes[g]) for g in bins], np.int64)
        keys = np.zeros((cnt, B.KEY_WORDS), np.int32)
        for g in range(nb):
            sel = np.nonzero(bins == g)[0]
            if len(sel):
                keys[sel] = gen_keys(kind, alphas[sel], sizes[g], prf, rng)[0]
        batches.append((keys, bins))
    update_after = 6                              # calls 0..5 see the old rows, 6.. the new ones
    ub = np.array([0, 1, 2, 3, 3], np.int32)
    ui = np.array([0, sizes[1] - 1, 7, 5, sizes[3] - 1], np.int64)
    rows = random_table(len(ub), e, seed=902)
    ctx = B.GroupContext(tables, **kw)
    try:
        want = [ctx.eval(k, b, prf) if i < update_after else None for i, (k, b) in enumerate(batches)]
        keys_dev = [torch.from_numpy(k).cuda() for k, _ in batches]
        outs = [torch.full((len(k), e), -1, dtype=torch.int32, device="cuda") for k, _ in batches]
        streams = [torch.cuda.Stream() for _ in range(nstreams)]
        torch.cuda.synchronize()
        host_mid = None
        for i, (k, b) in enumerate(batches):
            if i == 3:                            # a host evaluation among the device calls
                host_mid = ctx.eval(batches[1][0], batches[1][1], prf)
            if i == update_after:                 # a row update among them
                ctx.update_rows(ub, ui, rows)
            ctx.eval_device(keys_dev[i].data_ptr(), b, prf, outs[i].data_ptr(), streams[i % nstreams].cuda_stream)
        torch.cuda.synchronize()
        for g, i, r in zip(ub, ui, rows):
            tables[g][i] = r
        assert np.array_equal(host_mid, want[1])
        for i, (k, b) in enumerate(batches):
            if want[i] is None:
                want[i] = ctx.eval(k, b, prf)
            assert np.array_equal(outs[i].cpu().numpy(), want[i]), i
        # the update reached the results of the later calls
        touched = [i for i in range(update_after, len(batches)) if np.isin(batches[i][1], ub).any()]
        assert touched
    finally:
        ctx.close()


def test_returns_while_stream_busy(torch_cuda):
    """the call enqueues and returns: its stream is still busy afterwards"""
    torch = torch_cuda
    prf, e = B.PRF_CHACHA20, 16
    kw, sizes = KINDS["xor"]
    ka, kb, bins, alphas = gen_pairs("xor", sizes, PER_BIN, prf, seed=950)
    tables = [random_table(n, e, seed=951 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **kw)
    try:
        want = ctx.eval(ka, bins, prf)
        keys_dev = torch.from_numpy(ka).cuda()
        out = torch.full((len(ka), e), -1, dtype=torch.int32, device="cuda")
        s = torch.cuda.Stream()
        ctx.eval_device(keys_dev.data_ptr(), bins, prf, out.data_ptr(), s.cuda_stream)   # buffers at full size
        s.synchronize()
        out.fill_(-1)
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            torch.cuda._sleep(1 << 29)            # about a quarter of a second
        ctx.eval_device(keys_dev.data_ptr(), bins, prf, out.data_ptr(), s.cuda_stream)
        assert not s.query()
        s.synchronize()
        assert np.array_equal(out.cpu().numpy(), want)
    finally:
        ctx.close()


def test_bins_past_4_gib(torch_cuda):
    """a 2^26-row first bin (4 GiB of 64-byte rows): the small bins' rows start past 4 GiB.  The big bin is
    zero except on its alphas, so every pair of every bin reconstructs its row."""
    torch = torch_cuda
    prf, e = B.PRF_AES128, 16
    sizes = [1 << 26, 256, 1 << 10, 1 << 14]
    need = sum(sizes) * 64 + (1 << 26) * e * 4
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    if free < need + 2 * GiB:
        pytest.skip("needs %.1f GiB of device memory, %.1f GiB free" % (need / GiB, free / GiB))
    ka, kb, bins, alphas = gen_pairs("xor", sizes, [5, 6, 7, 6], prf, seed=600)
    support = np.unique(alphas[bins == 0])
    big = S.host_table(sizes[0], support, S.values(len(support), e, seed=7))
    small = [random_table(n, e, seed=610 + g) for g, n in enumerate(sizes[1:])]
    tables = [big] + small
    ctx = B.GroupContext(tables, xor=True)
    try:
        check_pairs(torch, "xor", ctx, tables, ka, kb, bins, alphas, prf)
    finally:
        ctx.close()
        del big, tables


@pytest.mark.parametrize("kind", list(KINDS))
def test_dpf_cpp_path(torch_cuda, kind):
    torch = torch_cuda
    import dpf
    cpp = dpf.dpf_cpp
    init = {"standard": cpp.group_init, "et": cpp.group_init_et, "xor": cpp.group_init_xor}[kind]
    prf = B.PRF_CHACHA20
    sizes = KINDS[kind][1][1:4]
    tables = [random_table(n, 16, seed=700 + g) for g, n in enumerate(sizes)]
    ka, kb, bins, alphas = gen_pairs(kind, sizes, [5, 5, 5], prf, seed=701)
    buf = init([torch.from_numpy(t) for t in tables], 0)
    try:
        res = []
        for k in (ka, kb):
            keys_dev = torch.from_numpy(k).cuda()
            out = torch.empty((len(k), 16), dtype=torch.int32, device="cuda")
            cpp.group_eval_device(keys_dev.data_ptr(), torch.from_numpy(bins), len(k), buf, prf, out.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream)
            res.append(out.cpu().numpy())
            assert np.array_equal(res[-1], cpp.group_eval(torch.from_numpy(k), torch.from_numpy(bins), buf, prf).numpy())
        assert np.array_equal(reconstruct(kind, *res), selected_rows(tables, bins, alphas))
        with pytest.raises(RuntimeError, match="group_eval_device: bins must be a CPU tensor"):
            cpp.group_eval_device(keys_dev.data_ptr(), torch.from_numpy(bins).cuda(), len(kb), buf, prf, out.data_ptr(), 0)
        with pytest.raises(RuntimeError, match="group_eval_device: bins must be a contiguous CPU int32"):
            cpp.group_eval_device(keys_dev.data_ptr(), torch.from_numpy(bins).long(), len(kb), buf, prf, out.data_ptr(), 0)
        with pytest.raises(RuntimeError, match=r"group_eval_device: .*bin 3 out of range"):
            cpp.group_eval_device(keys_dev.data_ptr(), torch.full((len(kb),), 3, dtype=torch.int32), len(kb), buf, prf,
                                  out.data_ptr(), 0)
    finally:
        cpp.eval_free(buf)


def test_binned_dpf(torch_cuda):
    torch = torch_cuda
    import dpf
    prf = B.PRF_AES128
    sizes = [2, 64, 1 << 10]
    tables = [random_table(n, 24, seed=710 + g) for g, n in enumerate(sizes)]
    ka, kb, bins, alphas = gen_pairs("standard", sizes, [4, 33, 6], prf, seed=711)
    d = dpf.BinnedDPF(prf=prf)
    d.eval_init([torch.from_numpy(t) for t in tables])
    try:
        ra = d.eval_gpu_device(torch.from_numpy(ka).cuda(), bins)            # numpy bins
        rb = torch.zeros((len(kb), 24), dtype=torch.int32, device="cuda")
        assert d.eval_gpu_device(torch.from_numpy(kb).cuda(), torch.from_numpy(bins), out_dev=rb) is rb
        torch.cuda.synchronize()
        ra, rb = ra.cpu().numpy(), rb.cpu().numpy()
        assert np.array_equal(ra, d.eval_gpu(torch.from_numpy(ka), bins).numpy())
        assert np.array_equal(rb, d.eval_gpu(torch.from_numpy(kb), bins).numpy())
        assert np.array_equal(reconstruct("standard", ra, rb), selected_rows(tables, bins, alphas))
        keys_dev = torch.from_numpy(ka).cuda()
        with pytest.raises(Exception, match="bins must be on the host.*synchronisation"):
            d.eval_gpu_device(keys_dev, torch.from_numpy(bins).cuda())
        with pytest.raises(Exception, match="keys_dev must be a contiguous int32 \\[B, 524\\] tensor on cuda:0"):
            d.eval_gpu_device(keys_dev[:, :500], bins)
        with pytest.raises(Exception, match="keys_dev must be"):
            d.eval_gpu_device(keys_dev.long(), bins)
        with pytest.raises(Exception, match="keys_dev must be"):
            d.eval_gpu_device(torch.from_numpy(ka), bins)                  # host keys
        with pytest.raises(Exception, match="one bin per key"):
            d.eval_gpu_device(keys_dev, bins[:-1])
        with pytest.raises(Exception, match="out_dev must be a contiguous int32"):
            d.eval_gpu_device(keys_dev, bins, out_dev=torch.zeros((len(ka), 23), dtype=torch.int32, device="cuda"))
        with pytest.raises(Exception, match="out_dev must be"):
            d.eval_gpu_device(keys_dev, bins, out_dev=torch.zeros((len(ka), 24), dtype=torch.int32))
    finally:
        d.close()


def test_group_context_refusals(torch_cuda):
    torch = torch_cuda
    prf = B.PRF_AES128
    tables = [random_table(n, 16, seed=720 + g) for g, n in enumerate([256, 1 << 10])]
    ka, _, bins, _ = gen_pairs("xor", [256, 1 << 10], [6, 6], prf, seed=721)
    ctx = B.GroupContext(tables, xor=True)
    plain = B.Context(tables[0], xor=True)
    try:
        want = ctx.eval(ka, bins, prf)
        keys_dev = torch.from_numpy(ka).cuda()
        out = torch.zeros((len(ka), 16), dtype=torch.int32, device="cuda")
        p, o = keys_dev.data_ptr(), out.data_ptr()
        for args, what in [((p, np.full(len(ka), 2, np.int32), prf, o), r"\(-1\).*key 0: bin 2 out of range"),
                           ((p, bins, 4, o), r"\(-1\).*unknown prf id 4"),
                           ((0, bins, prf, o), r"\(-1\).*null buffer"),
                           ((p, bins, prf, 0), r"\(-1\).*null buffer"),
                           ((p, bins[:0], prf, o), r"\(-1\).*nkeys=0 out of range"),
                           ((p + 4, bins, prf, o), r"\(-1\).*16-byte aligned"),
                           ((p, bins, prf, o + 2), r"\(-1\).*aligned")]:
            with pytest.raises(B.B200DPFError, match=what):
                ctx.eval_device(*args)
        with pytest.raises(B.B200DPFError, match=r"b200dpf_group_eval_device failed \(-4\).*not a grouped context"):
            B.GroupContext.eval_device(plain, p, bins, prf, o)
        torch.cuda.synchronize()
        assert not out.any()                      # nothing was enqueued
        assert np.array_equal(device_eval(torch, ctx, ka, bins, prf), want)
    finally:
        ctx.close()
        plain.close()
