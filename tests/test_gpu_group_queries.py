"""Batch-PIR query batches on the GPU (b200dpf_group_eval_queries_device): Q queries of one key per bin, wire
format or compact queries, from device memory into device results, for all three kinds of key.  Every result is
compared bit for bit with b200dpf_group_eval_device on the same keys with the bins 0 .. nbins-1 tiled Q times,
and every pair reconstructs its row (a - b, or a ^ b, = table[g][alpha]); some cases are also checked against
b200dpf_group_eval and some pairs against the per-index oracles.  Also covered: the cached plan (the same Q
twice, Q changing and coming back, the prf alternating, an option set, other grouped evaluations in between),
back-to-back calls on one and two streams with a row update among them, a repeated shape that returns while
its stream is busy, 1,024 bins x 64 queries, a bin whose successors start past 4 GiB, and the three Python
layers."""
import ctypes as C
import os
import re
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
import oracle  # noqa: E402
import sparse_oracle as S  # noqa: E402
import xor_oracle  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
ES = [1, 5, 16, 33, 40]
QS = [1, 3, 33, 70]
GiB = 1 << 30

# per kind: GroupContext keyword, dpf_cpp initialiser, bin sizes of mixed depths (from the smallest the kind takes)
KINDS = {
    "standard": ({}, "group_init", [2, 64, 1 << 10, 8, 1 << 14]),
    "et": ({"early_termination": True}, "group_init_et", [8, 1 << 12, 64, 1 << 14, 1 << 10]),
    "xor": ({"xor": True}, "group_init_xor", [256, 1 << 14, 512, 1 << 10, 1 << 12]),
}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


@pytest.fixture(scope="module")
def orc():
    return oracle.Oracle()


def gen_keys(kind, alphas, n, prf, rng):
    if kind == "standard":
        return B.gen_batch(alphas, n, rng.randint(0, 2**31, size=len(alphas)), prf)
    seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
    return (B.gen_batch_et if kind == "et" else B.gen_batch_xor)(alphas, n, seeds, prf)


def gen_queries(kind, sizes, nq, prf, seed):
    """nq queries of one key pair per bin: int32 [nq, nbins, 524] twice, and the alphas [nq, nbins] (each
    bin's first and last row among them)"""
    rng = np.random.RandomState(seed)
    ka = np.zeros((nq, len(sizes), B.KEY_WORDS), np.int32)
    kb = np.zeros_like(ka)
    alphas = np.zeros((nq, len(sizes)), np.int64)
    for g, n in enumerate(sizes):
        al = rng.randint(0, n, size=nq).astype(np.int64)
        al[:2] = [0, n - 1][:nq]
        ka[:, g], kb[:, g] = gen_keys(kind, al, n, prf, rng)
        alphas[:, g] = al
    return ka, kb, alphas


def tiled_bins(nq, nbins):
    return np.tile(np.arange(nbins, dtype=np.int32), nq)


def reconstruct(kind, a, b):
    if kind == "xor":
        return (a.view(np.uint32) ^ b.view(np.uint32)).view(np.int32)
    return (a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32)


def selected_rows(tables, alphas):
    return np.stack([np.stack([tables[g][a] for g, a in enumerate(row)]) for row in alphas])


def upload(torch, ctx, keys, compact):
    return torch.from_numpy(ctx.pack_queries(keys) if compact else np.ascontiguousarray(keys)).cuda()


def queries_eval(torch, ctx, keys, prf, compact, stream=None):
    """GroupContext.eval_queries_device on keys uploaded with torch; int32 [Q, nbins, E] back on the host"""
    keys_dev = upload(torch, ctx, keys, compact)
    out = torch.full((keys.shape[0], ctx.nbins, ctx.entry_size), -1, dtype=torch.int32, device="cuda")
    st = stream if stream is not None else torch.cuda.current_stream()
    ctx.eval_queries_device(keys_dev.data_ptr(), keys.shape[0], prf, out.data_ptr(), st.cuda_stream, compact=compact)
    st.synchronize()
    return out.cpu().numpy()


def device_ref(torch, ctx, keys, prf):
    """b200dpf_group_eval_device on the same keys with tiled bins, as [Q, nbins, E]"""
    nq, nbins = keys.shape[:2]
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys.reshape(-1, B.KEY_WORDS))).cuda()
    out = torch.full((nq * nbins, ctx.entry_size), -1, dtype=torch.int32, device="cuda")
    ctx.eval_device(keys_dev.data_ptr(), tiled_bins(nq, nbins), prf, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(nq, nbins, ctx.entry_size)


def oracle_rows(orc, kind, keys, prf, table):
    """the per-index oracle of the kind: int32 [len(keys), E]"""
    if kind == "standard":
        return orc.eval_dot(keys, prf, table)
    if kind == "et":
        return et_oracle.dot_u32(np.stack([et_oracle.eval_full_flat_et(orc, k, prf) for k in keys]), table)
    return xor_oracle.eval_xor(orc, keys, prf, table)


def make_context(kind, sizes, e, seed):
    tables = [random_table(n, e, seed=seed + g) for g, n in enumerate(sizes)]
    return B.GroupContext(tables, **KINDS[kind][0]), tables


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("e", ES)
@pytest.mark.parametrize("kind", list(KINDS))
def test_queries_bit_exact(torch_cuda, orc, kind, e, prf):
    """both formats against the device path with tiled bins, the pairs reconstructing their rows"""
    torch = torch_cuda
    sizes = KINDS[kind][2]
    nq = QS[(ES.index(e) + prf) % len(QS)]
    ka, kb, alphas = gen_queries(kind, sizes, nq, prf, seed=100 + 7 * prf + e)
    ctx, tables = make_context(kind, sizes, e, seed=10 * e)
    try:
        want_a, want_b = device_ref(torch, ctx, ka, prf), device_ref(torch, ctx, kb, prf)
        assert np.array_equal(reconstruct(kind, want_a, want_b), selected_rows(tables, alphas))
        for compact in (False, True):
            ra = queries_eval(torch, ctx, ka, prf, compact)
            assert ctx.last_launches == (e + 15) // 16            # the evaluation launches, timed alone
            assert ctx.last_device_ms > 0
            rb = queries_eval(torch, ctx, kb, prf, compact)
            assert np.array_equal(ra, want_a), compact
            assert np.array_equal(rb, want_b), compact
        if e == 16:                               # the host path
            assert np.array_equal(want_a.reshape(-1, e), ctx.eval(ka.reshape(-1, B.KEY_WORDS), tiled_bins(nq, len(sizes)), prf))
        if e == 5:                                # the per-index oracle, query 0 of every bin
            for g, t in enumerate(tables):
                assert np.array_equal(ra[0, g:g + 1], oracle_rows(orc, kind, ka[0, g:g + 1], prf, t)), g
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_plan_cache(torch_cuda, kind):
    """the cached plan stays right when Q, the prf or an option changes, and when other grouped evaluations,
    which upload lists of their own, run between two cached calls"""
    torch = torch_cuda
    sizes = KINDS[kind][2]
    e = 20
    ctx, tables = make_context(kind, sizes, e, seed=400)
    keys = {prf: gen_queries(kind, sizes, 70, prf, seed=401 + prf) for prf in (B.PRF_CHACHA20, B.PRF_AES128)}
    try:
        def check(nq, prf, compact):
            ka, kb, alphas = keys[prf]
            ra = queries_eval(torch, ctx, ka[:nq], prf, compact)
            rb = queries_eval(torch, ctx, kb[:nq], prf, compact)
            assert np.array_equal(ra, device_ref(torch, ctx, ka[:nq], prf)), (nq, prf, compact)
            assert np.array_equal(reconstruct(kind, ra, rb), selected_rows(tables, alphas[:nq])), (nq, prf, compact)

        aes, chacha = B.PRF_AES128, B.PRF_CHACHA20
        check(70, aes, False)
        check(70, aes, False)                     # the same Q twice
        check(1, aes, True)                       # 70 -> 1 -> 70
        check(70, aes, True)
        for prf in (chacha, aes, chacha, aes):    # the same Q, the prf alternating
            check(70, prf, prf == aes)
        ctx.set_option("subtree_log2", 1)         # an option between two same-Q calls
        check(70, aes, False)
        ctx.set_subtree_log2(0)
        check(70, aes, True)
        ka, _, _ = keys[aes]
        check(33, aes, False)
        mixed_bins = np.arange(len(sizes), dtype=np.int32)[::-1].copy()
        host = ctx.eval(ka[0][::-1].copy(), mixed_bins, aes)       # other grouped evaluations in between
        check(33, aes, True)
        keys_dev = torch.from_numpy(ka[0][::-1].copy()).cuda()
        out = torch.zeros((len(sizes), e), dtype=torch.int32, device="cuda")
        ctx.eval_device(keys_dev.data_ptr(), mixed_bins, aes, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
        check(33, aes, False)
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), host)
    finally:
        ctx.close()


@pytest.mark.parametrize("nstreams", [1, 2])
@pytest.mark.parametrize("kind", list(KINDS))
def test_back_to_back_without_syncs(torch_cuda, kind, nstreams):
    """ten calls with no synchronisation in between, of both formats and changing Q, with a row update among
    them: calls before it see the old rows and calls after it the new ones"""
    torch = torch_cuda
    prf, e = B.PRF_AES128, 20
    sizes = KINDS[kind][2]
    ctx, tables = make_context(kind, sizes, e, seed=900)
    counts = [3, 3, 33, 1, 70, 70, 3, 33, 33, 70]
    batches = [gen_queries(kind, sizes, nq, prf, seed=901 + i)[0] for i, nq in enumerate(counts)]
    update_after = 6
    ub = np.array([0, 1, 2, 3, 4], np.int32)
    ui = np.array([0, sizes[1] - 1, 1, 5, sizes[4] - 1], np.int64)
    rows = random_table(len(ub), e, seed=902)
    try:
        old = [device_ref(torch, ctx, k, prf) for k in batches]
        keys_dev = [upload(torch, ctx, k, i % 2 == 1) for i, k in enumerate(batches)]
        outs = [torch.full((nq, len(sizes), e), -1, dtype=torch.int32, device="cuda") for nq in counts]
        streams = [torch.cuda.Stream() for _ in range(nstreams)]
        torch.cuda.synchronize()
        for i, nq in enumerate(counts):
            if i == update_after:
                ctx.update_rows(ub, ui, rows)
            ctx.eval_queries_device(keys_dev[i].data_ptr(), nq, prf, outs[i].data_ptr(), streams[i % nstreams].cuda_stream,
                                    compact=i % 2 == 1)
        torch.cuda.synchronize()
        changed = np.zeros(len(sizes), bool)
        for i, k in enumerate(batches):
            got = outs[i].cpu().numpy()
            if i < update_after:
                assert np.array_equal(got, old[i]), i
            else:
                new = device_ref(torch, ctx, k, prf)
                assert np.array_equal(got, new), i
                changed |= (new != old[i]).any(axis=(0, 2))
        assert changed.all()                      # the later calls saw the new rows of every bin
    finally:
        ctx.close()


def test_repeated_shape_returns_while_stream_busy(torch_cuda):
    """a call of the previous call's shape only enqueues: its stream is still busy when it returns"""
    torch = torch_cuda
    prf, e, nq = B.PRF_CHACHA20, 16, 33
    sizes = KINDS["xor"][2]
    ka, _, _ = gen_queries("xor", sizes, nq, prf, seed=950)
    ctx, _ = make_context("xor", sizes, e, seed=951)
    try:
        want = device_ref(torch, ctx, ka, prf)
        wire, packed = upload(torch, ctx, ka, False), upload(torch, ctx, ka, True)
        out = torch.full((nq, len(sizes), e), -1, dtype=torch.int32, device="cuda")
        s = torch.cuda.Stream()
        ctx.eval_queries_device(wire.data_ptr(), nq, prf, out.data_ptr(), s.cuda_stream)     # plans this shape
        s.synchronize()
        for keys_dev, compact in ((wire, False), (packed, True)):
            out.fill_(-1)
            torch.cuda.synchronize()
            with torch.cuda.stream(s):
                torch.cuda._sleep(1 << 29)        # about a quarter of a second
            ctx.eval_queries_device(keys_dev.data_ptr(), nq, prf, out.data_ptr(), s.cuda_stream, compact=compact)
            assert not s.query(), compact
            s.synchronize()
            assert np.array_equal(out.cpu().numpy(), want), compact
    finally:
        ctx.close()


def test_1024_bins_64_queries(torch_cuda):
    """65,536 XOR-shared pairs: 1,024 bins of 2^10 rows, 64 queries"""
    torch = torch_cuda
    prf, e, nq = B.PRF_AES128, 16, 64
    sizes = [1 << 10] * 1024
    ka, kb, alphas = gen_queries("xor", sizes, nq, prf, seed=960)
    ctx, tables = make_context("xor", sizes, e, seed=961)
    try:
        assert ctx.query_bytes == 1024 * 224
        ra = queries_eval(torch, ctx, ka, prf, True)
        rb = queries_eval(torch, ctx, kb, prf, False)
        assert np.array_equal(ra, device_ref(torch, ctx, ka, prf))
        assert np.array_equal(reconstruct("xor", ra, rb), selected_rows(tables, alphas))
    finally:
        ctx.close()


def test_bins_past_4_gib(torch_cuda):
    """a 2^26-row first bin (4 GiB of 64-byte rows): the small bins' rows start past 4 GiB.  The big bin is
    zero except on its alphas, so every pair of every bin reconstructs its row."""
    torch = torch_cuda
    prf, e, nq = B.PRF_AES128, 16, 3
    sizes = [1 << 26, 256, 1 << 10, 1 << 14]
    need = sum(sizes) * 64 + (1 << 26) * e * 4
    torch.cuda.synchronize()
    free, _ = torch.cuda.mem_get_info()
    if free < need + 2 * GiB:
        pytest.skip("needs %.1f GiB of device memory, %.1f GiB free" % (need / GiB, free / GiB))
    ka, kb, alphas = gen_queries("xor", sizes, nq, prf, seed=970)
    support = np.unique(alphas[:, 0])
    big = S.host_table(sizes[0], support, S.values(len(support), e, seed=7))
    tables = [big] + [random_table(n, e, seed=971 + g) for g, n in enumerate(sizes[1:])]
    ctx = B.GroupContext(tables, xor=True)
    try:
        for compact in (False, True):
            ra = queries_eval(torch, ctx, ka, prf, compact)
            rb = queries_eval(torch, ctx, kb, prf, not compact)
            assert np.array_equal(ra, device_ref(torch, ctx, ka, prf)), compact
            assert np.array_equal(reconstruct("xor", ra, rb), selected_rows(tables, alphas)), compact
    finally:
        ctx.close()
        del big, tables


@pytest.mark.parametrize("kind", list(KINDS))
def test_dpf_cpp_path(torch_cuda, kind):
    torch = torch_cuda
    import dpf
    cpp = dpf.dpf_cpp
    prf, e, nq = B.PRF_CHACHA20, 16, 5
    sizes = KINDS[kind][2][:4]
    tables = [random_table(n, e, seed=700 + g) for g, n in enumerate(sizes)]
    ka, kb, alphas = gen_queries(kind, sizes, nq, prf, seed=701)
    buf = getattr(cpp, KINDS[kind][1])([torch.from_numpy(t) for t in tables], 0)
    packer = B.GroupContext.__new__(B.GroupContext)     # pack_queries needs only the kind and the bin sizes
    packer.kind, packer.tables = {"standard": "", "et": "_et", "xor": "_xor"}[kind], tables
    try:
        assert cpp.group_query_bytes(buf) == sum(len(B._key_pack(packer.kind, ka[0, g])) for g in range(len(sizes)))
        bins = torch.from_numpy(tiled_bins(nq, len(sizes)))
        res = []
        for keys, compact in ((ka, True), (kb, False)):
            keys_dev = torch.from_numpy(packer.pack_queries(keys) if compact else keys).cuda()
            out = torch.empty((nq, len(sizes), e), dtype=torch.int32, device="cuda")
            cpp.group_eval_queries_device(keys_dev.data_ptr(), nq, buf, prf, out.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream, compact)
            res.append(out.cpu().numpy())
            want = cpp.group_eval(torch.from_numpy(keys.reshape(-1, B.KEY_WORDS)), bins, buf, prf).numpy()
            assert np.array_equal(res[-1].reshape(-1, e), want)
        assert np.array_equal(reconstruct(kind, *res), selected_rows(tables, alphas))
        with pytest.raises(RuntimeError, match=r"group_eval_queries_device: .*nqueries=0 out of range"):
            cpp.group_eval_queries_device(keys_dev.data_ptr(), 0, buf, prf, out.data_ptr(), 0, False)
    finally:
        cpp.eval_free(buf)


def test_binned_dpf(torch_cuda):
    torch = torch_cuda
    import dpf
    prf, e, nq = B.PRF_AES128, 24, 6
    sizes = [2, 64, 1 << 10]
    tables = [random_table(n, e, seed=710 + g) for g, n in enumerate(sizes)]
    ka, kb, alphas = gen_queries("standard", sizes, nq, prf, seed=711)
    d = dpf.BinnedDPF(prf=prf)
    d.eval_init([torch.from_numpy(t) for t in tables])
    try:
        packed = np.stack([np.frombuffer(b"".join(B.key_pack(k) for k in q), np.uint8) for q in kb])
        ra = d.eval_queries_device(torch.from_numpy(ka).cuda())
        rb = torch.zeros((nq, len(sizes), e), dtype=torch.int32, device="cuda")
        assert d.eval_queries_device(torch.from_numpy(packed).cuda(), out_dev=rb) is rb
        torch.cuda.synchronize()
        ra, rb = ra.cpu().numpy(), rb.cpu().numpy()
        bins = tiled_bins(nq, len(sizes))
        assert np.array_equal(ra.reshape(-1, e), d.eval_gpu(torch.from_numpy(ka.reshape(-1, B.KEY_WORDS)), bins).numpy())
        assert np.array_equal(rb.reshape(-1, e), d.eval_gpu(torch.from_numpy(kb.reshape(-1, B.KEY_WORDS)), bins).numpy())
        assert np.array_equal(reconstruct("standard", ra, rb), selected_rows(tables, alphas))
        keys_dev, packed_dev = torch.from_numpy(ka).cuda(), torch.from_numpy(packed).cuda()
        with pytest.raises(Exception, match=r"int32 keys_dev must be \[Q, 3, 524\]"):
            d.eval_queries_device(keys_dev[:, :2].contiguous())
        with pytest.raises(Exception, match=r"uint8 keys_dev must be \[Q, %d\]" % packed.shape[1]):
            d.eval_queries_device(packed_dev[:, 16:].contiguous())
        with pytest.raises(Exception, match=r"keys_dev must be a contiguous CUDA tensor on cuda:0"):
            d.eval_queries_device(keys_dev.long())
        with pytest.raises(Exception, match=r"keys_dev must be a contiguous CUDA tensor"):
            d.eval_queries_device(torch.from_numpy(ka))                       # host keys
        with pytest.raises(Exception, match=r"out_dev must be a contiguous int32 \[6, 3, 24\]"):
            d.eval_queries_device(keys_dev, out_dev=torch.zeros((nq, 3, 23), dtype=torch.int32, device="cuda"))
        with pytest.raises(Exception, match=r"out_dev must be"):
            d.eval_queries_device(keys_dev, out_dev=torch.zeros((nq, 3, 24), dtype=torch.int32))
    finally:
        d.close()


def test_group_context_refusals(torch_cuda):
    torch = torch_cuda
    prf, nq = B.PRF_AES128, 4
    sizes = [256, 1 << 10]
    ka, _, _ = gen_queries("xor", sizes, nq, prf, seed=721)
    ctx, _ = make_context("xor", sizes, 16, seed=720)
    plain = B.Context(random_table(256, 16, seed=722), xor=True)
    try:
        want = device_ref(torch, ctx, ka, prf)
        keys_dev = torch.from_numpy(ka).cuda()
        out = torch.zeros((nq, 2, 16), dtype=torch.int32, device="cuda")
        p, o = keys_dev.data_ptr(), out.data_ptr()
        L = B.lib()
        for args, what in [((p, B.KEYS_WIRE, 0, prf, o), r"nqueries=0 out of range"),
                           ((p, B.KEYS_WIRE, (1 << 23) + 1, prf, o), r"nqueries=8388609 out of range"),
                           ((p, 2, nq, prf, o), r"unknown key_format 2"),
                           ((p, -1, nq, prf, o), r"unknown key_format -1"),
                           ((p, B.KEYS_COMPACT, nq, 4, o), r"unknown prf id 4"),
                           ((0, B.KEYS_WIRE, nq, prf, o), r"null buffer"),
                           ((p, B.KEYS_WIRE, nq, prf, 0), r"null buffer"),
                           ((p + 4, B.KEYS_COMPACT, nq, prf, o), r"16-byte aligned"),
                           ((p, B.KEYS_WIRE, nq, prf, o + 2), r"aligned")]:
            k, fmt, n, pr, out_ptr = args
            assert L.b200dpf_group_eval_queries_device(ctx.handle, C.c_void_p(k), fmt, n, pr, C.c_void_p(out_ptr), None) == -1
            assert re.search(what, L.b200dpf_last_error().decode()), what
        with pytest.raises(B.B200DPFError, match=r"b200dpf_group_eval_queries_device failed \(-4\).*not a grouped context"):
            B.GroupContext.eval_queries_device(plain, p, nq, prf, o)
        assert L.b200dpf_group_query_bytes(plain.handle) == -1
        torch.cuda.synchronize()
        assert not out.any()                      # nothing was enqueued
        assert np.array_equal(queries_eval(torch, ctx, ka, prf, False), want)
    finally:
        ctx.close()
        plain.close()
