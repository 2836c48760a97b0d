"""GPU key generation for every kind of key: b200dpf_gen_batch_gpu_et / _xor against the CPU's gen_batch_et /
_xor at every depth, and batch-PIR query batches made on the GPU (b200dpf_group_gen_queries_device) against the
host keys of each (query, bin) pair and pack_queries of them, byte for byte, for both servers and both formats.
Also: generated queries evaluated on the same stream with no sync in between (and at one throughput shape per
kind), alphas taken mod the bin size, the order of the per-bin table's upload against a first call on another
stream, the cached plan left alone by a generator call, and the Python layers."""
import ctypes as C
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
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
QS = (1, 3, 33, 256)
SENTINEL = 0xA5

# per kind: GroupContext keyword, KINDS suffix, bin sizes of mixed depths (those of test_group_queries_host.py)
KINDS = {
    "standard": ({}, "", [2, 64, 1 << 10, 8]),
    "et": ({"early_termination": True}, "_et", [8, 64, 1 << 10, 32]),
    "xor": ({"xor": True}, "_xor", [256, 1 << 12, 512, 1 << 10]),
}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


def host_gen(suffix, alphas, n, seeds, prf):
    """the CPU's ChaCha20-DRBG keygen of the kind"""
    return getattr(B, "gen_batch_secure" if suffix == "" else "gen_batch" + suffix)(alphas, n, seeds, prf)


def host_queries(ctx, alphas, seeds, prf):
    """int32 [Q, nbins, 524] twice: key (q, g) from gen_batch<kind>(alphas[q, g] mod n_g, n_g, seeds[q, g])"""
    nq, nbins = alphas.shape
    ka = np.zeros((nq, nbins, B.KEY_WORDS), np.int32)
    kb = np.zeros_like(ka)
    for g, t in enumerate(ctx.tables):
        n = t.shape[0]
        ka[:, g], kb[:, g] = host_gen(ctx.kind, alphas[:, g] % n, n, seeds[:, g].tobytes(), prf)
    return ka, kb


def random_queries(ctx, nq, seed):
    rng = np.random.RandomState(seed)
    sizes = [t.shape[0] for t in ctx.tables]
    alphas = np.stack([rng.randint(0, n, size=nq) for n in sizes], axis=1).astype(np.int64)
    alphas[0] = 0
    if nq > 1:
        alphas[1] = [n - 1 for n in sizes]
    return alphas, rng.randint(0, 256, size=(nq, len(sizes), 44)).astype(np.uint8)


def gen_device(torch, ctx, alphas, seeds, prf, compact, stream=None, sentinel=64):
    """GroupContext.gen_queries_device into buffers with `sentinel` bytes of SENTINEL after the last query;
    both outputs as host bytes, the sentinels checked"""
    nq, nbins = alphas.shape
    size = nq * (ctx.query_bytes if compact else nbins * B.KEY_WORDS * 4)
    outs = [torch.full((size + sentinel,), SENTINEL, dtype=torch.uint8, device="cuda") for _ in range(2)]
    st = stream if stream is not None else torch.cuda.current_stream()
    with torch.cuda.stream(st):
        a_dev = torch.from_numpy(alphas).cuda()
        s_dev = torch.from_numpy(np.ascontiguousarray(seeds)).cuda()
    ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, prf, outs[0].data_ptr(), outs[1].data_ptr(),
                           st.cuda_stream, compact=compact)
    st.synchronize()
    res = []
    for o in outs:
        h = o.cpu().numpy()
        assert (h[size:] == SENTINEL).all(), "bytes after the last query written"
        res.append(h[:size])
    return res


def reconstruct(kind, a, b):
    if kind == "xor":
        return (a.view(np.uint32) ^ b.view(np.uint32)).view(np.int32)
    return (a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32)


def selected_rows(tables, alphas):
    return np.stack([np.stack([tables[g][a % len(tables[g])] for g, a in enumerate(row)]) for row in alphas])


def make_context(kind, sizes, e, seed):
    tables = [random_table(n, e, seed=seed + g) for g, n in enumerate(sizes)]
    return B.GroupContext(tables, **KINDS[kind][0]), tables


# ---- b200dpf_gen_batch_gpu_et / _xor ----------------------------------------------------------------------

@pytest.mark.parametrize("suffix,max_depth,lane_bits", [("_et", 29, 2), ("_xor", 24, 7)])
@pytest.mark.parametrize("prf", PRFS)
def test_gen_batch_gpu_kind_every_depth(torch_cuda, suffix, max_depth, lane_bits, prf):
    """byte-identical to gen_batch_et / _xor at every depth of the kind, at alpha 0, n - 1 and the lane edges,
    into host and device memory"""
    torch = torch_cuda
    rng = np.random.RandomState(prf * 100 + lane_bits)
    gpu = getattr(B, "gen_batch_gpu" + suffix)
    edges = (0, 3) if lane_bits == 2 else (0, 31, 32, 127)
    for depth in range(1, max_depth + 1):
        n = 1 << (depth + lane_bits)
        leaves = rng.randint(0, 1 << depth, size=2)
        alphas = np.array([0, n - 1] + [(int(v) << lane_bits) | e for v in leaves for e in edges], np.int64)
        seeds = rng.bytes(44 * len(alphas))
        ha, hb = host_gen(suffix, alphas, n, seeds, prf)
        ga, gb = gpu(alphas, n, seeds, prf)
        assert np.array_equal(ga, ha) and np.array_equal(gb, hb), depth
        da = torch.full((len(alphas), B.KEY_WORDS), -1, dtype=torch.int32, device="cuda")
        db = torch.full_like(da, -1)
        gpu(alphas, n, seeds, prf, out_ptrs=(da.data_ptr(), db.data_ptr()))
        torch.cuda.synchronize()
        assert np.array_equal(da.cpu().numpy(), ha) and np.array_equal(db.cpu().numpy(), hb), depth


# ---- b200dpf_group_gen_queries_device ---------------------------------------------------------------------

@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("prf", PRFS)
def test_queries_match_host_keys(torch_cuda, kind, prf):
    """wire output = the host keys of every (query, bin) pair, all 524 words; compact output = pack_queries of
    them; both servers; nothing written after the last query"""
    torch = torch_cuda
    ctx, _ = make_context(kind, KINDS[kind][2], 1, 10 + prf)
    for nq in QS:
        alphas, seeds = random_queries(ctx, nq, 1000 * prf + nq)
        ka, kb = host_queries(ctx, alphas, seeds, prf)
        wa, wb = gen_device(torch, ctx, alphas, seeds, prf, compact=False)
        assert np.array_equal(wa.view(np.int32).reshape(ka.shape), ka), (kind, prf, nq)
        assert np.array_equal(wb.view(np.int32).reshape(kb.shape), kb), (kind, prf, nq)
        pa, pb = gen_device(torch, ctx, alphas, seeds, prf, compact=True)
        assert np.array_equal(pa.reshape(nq, -1), ctx.pack_queries(ka)), (kind, prf, nq)
        assert np.array_equal(pb.reshape(nq, -1), ctx.pack_queries(kb)), (kind, prf, nq)
    ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_alpha_taken_mod_bin_size(torch_cuda, kind):
    """out-of-range and negative alphas give the bytes of alpha mod n_g"""
    torch = torch_cuda
    ctx, _ = make_context(kind, KINDS[kind][2], 1, 20)
    alphas, seeds = random_queries(ctx, 6, 21)
    sizes = np.array([t.shape[0] for t in ctx.tables], np.int64)
    wild = alphas + np.array([[0], [1], [-1], [1 << 20], [-(1 << 40)], [0]], np.int64) * sizes
    wild[5] = np.iinfo(np.int64).min + alphas[5]            # -2^63 is a multiple of every bin size
    for compact in (False, True):
        want = gen_device(torch, ctx, alphas, seeds, B.PRF_AES128, compact)
        got = gen_device(torch, ctx, wild, seeds, B.PRF_AES128, compact)
        assert all(np.array_equal(w, g) for w, g in zip(want, got)), (kind, compact)
    ka, _ = host_queries(ctx, wild, seeds, B.PRF_AES128)
    wa, _ = gen_device(torch, ctx, wild, seeds, B.PRF_AES128, compact=False)
    assert np.array_equal(wa.view(np.int32).reshape(ka.shape), ka)
    ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("compact", [False, True])
def test_generate_then_evaluate_on_one_stream(torch_cuda, kind, compact):
    """generated queries go into eval_queries_device on the same non-default stream with no sync in between,
    for every PRF, and every pair reconstructs table[g][alpha mod n_g]"""
    torch = torch_cuda
    ctx, tables = make_context(kind, KINDS[kind][2], 5, 30)
    nq, nbins = 33, ctx.nbins
    st = torch.cuda.Stream()
    for prf in PRFS:
        alphas, seeds = random_queries(ctx, nq, 40 + prf)
        alphas[2:] += np.random.RandomState(prf).randint(-3, 3, size=alphas[2:].shape) * np.array([t.shape[0] for t in tables])
        size = nq * ctx.query_bytes if compact else nq * nbins * B.KEY_WORDS * 4
        with torch.cuda.stream(st):
            a_dev = torch.from_numpy(alphas).cuda()
            s_dev = torch.from_numpy(seeds).cuda()
            qa = torch.empty(size, dtype=torch.uint8, device="cuda")
            qb = torch.empty_like(qa)
            outs = [torch.full((nq, nbins, ctx.entry_size), -1, dtype=torch.int32, device="cuda") for _ in range(2)]
        ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, prf, qa.data_ptr(), qb.data_ptr(), st.cuda_stream,
                               compact=compact)
        for q, o in zip((qa, qb), outs):
            ctx.eval_queries_device(q.data_ptr(), nq, prf, o.data_ptr(), st.cuda_stream, compact=compact)
        st.synchronize()
        rec = reconstruct(kind, outs[0].cpu().numpy(), outs[1].cpu().numpy())
        assert np.array_equal(rec, selected_rows(tables, alphas)), (kind, prf)
    ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_throughput_shape_reconstructs(torch_cuda, kind):
    """256 bins of 2^10 rows x 256 queries (65,536 pairs), AES, compact: generate fresh queries twice on one
    stream and evaluate each batch; every pair reconstructs"""
    torch = torch_cuda
    nbins, n, nq, e = 256, 1 << 10, 256, 4
    ctx, tables = make_context(kind, [n] * nbins, e, 50)
    st = torch.cuda.Stream()
    g = torch.Generator(device="cuda").manual_seed(7)
    with torch.cuda.stream(st):
        qa = torch.empty(nq * ctx.query_bytes, dtype=torch.uint8, device="cuda")
        qb = torch.empty_like(qa)
        oa = torch.empty((nq, nbins, e), dtype=torch.int32, device="cuda")
        ob = torch.empty_like(oa)
        for rnd in range(2):
            alphas = torch.randint(0, n, (nq, nbins), dtype=torch.int64, device="cuda", generator=g)
            seeds = torch.randint(0, 256, (nq, nbins, 44), dtype=torch.uint8, device="cuda", generator=g)
            ctx.gen_queries_device(alphas.data_ptr(), seeds.data_ptr(), nq, B.PRF_AES128, qa.data_ptr(), qb.data_ptr(),
                                   st.cuda_stream, compact=True)
            ctx.eval_queries_device(qa.data_ptr(), nq, B.PRF_AES128, oa.data_ptr(), st.cuda_stream, compact=True)
            ctx.eval_queries_device(qb.data_ptr(), nq, B.PRF_AES128, ob.data_ptr(), st.cuda_stream, compact=True)
            st.synchronize()
            rec = reconstruct(kind, oa.cpu().numpy(), ob.cpu().numpy())
            assert np.array_equal(rec, selected_rows(tables, alphas.cpu().numpy())), (kind, rnd)
    ctx.close()


# ---- ordering ---------------------------------------------------------------------------------------------

def busy(torch, stream):
    """keep `stream` busy for a few milliseconds, so that whatever follows on it runs late"""
    with torch.cuda.stream(stream):
        torch.cuda._sleep(20_000_000)


@pytest.mark.parametrize("kind", list(KINDS))
def test_first_call_generates_then_other_stream_evaluates(torch_cuda, kind):
    """a fresh context whose first call is gen_queries_device on a busy stream S1 (so its upload of the per-bin
    table runs late), then eval_queries_device of compact queries made on the host, on S2 with no wait on S1:
    the evaluation must still read the complete table"""
    torch = torch_cuda
    ctx, tables = make_context(kind, KINDS[kind][2], 3, 60)
    nq = 3
    alphas, seeds = random_queries(ctx, nq, 61)
    ka, kb = host_queries(ctx, alphas, seeds, B.PRF_AES128)
    pa = torch.from_numpy(ctx.pack_queries(ka)).cuda()
    pb = torch.from_numpy(ctx.pack_queries(kb)).cuda()
    a_dev, s_dev = torch.from_numpy(alphas).cuda(), torch.from_numpy(seeds).cuda()
    qa = torch.empty(nq * ctx.query_bytes, dtype=torch.uint8, device="cuda")
    qb = torch.empty_like(qa)
    outs = [torch.full((nq, ctx.nbins, 3), -1, dtype=torch.int32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    busy(torch, s1)
    ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, B.PRF_AES128, qa.data_ptr(), qb.data_ptr(),
                           s1.cuda_stream, compact=True)
    for p, o in zip((pa, pb), outs):
        ctx.eval_queries_device(p.data_ptr(), nq, B.PRF_AES128, o.data_ptr(), s2.cuda_stream, compact=True)
    torch.cuda.synchronize()
    rec = reconstruct(kind, outs[0].cpu().numpy(), outs[1].cpu().numpy())
    assert np.array_equal(rec, selected_rows(tables, alphas))
    assert np.array_equal(qa.cpu().numpy().reshape(nq, -1), ctx.pack_queries(ka))
    ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_first_call_evaluates_then_other_stream_generates(torch_cuda, kind):
    """the reverse order: eval_queries_device of compact queries on a busy S1 first, then gen_queries_device on
    S2 with no wait on S1; the generated bytes are the host's"""
    torch = torch_cuda
    ctx, tables = make_context(kind, KINDS[kind][2], 3, 70)
    nq = 3
    alphas, seeds = random_queries(ctx, nq, 71)
    ka, kb = host_queries(ctx, alphas, seeds, B.PRF_AES128)
    pa = torch.from_numpy(ctx.pack_queries(ka)).cuda()
    out = torch.full((nq, ctx.nbins, 3), -1, dtype=torch.int32, device="cuda")
    a_dev, s_dev = torch.from_numpy(alphas).cuda(), torch.from_numpy(seeds).cuda()
    qa = torch.empty(nq * ctx.query_bytes, dtype=torch.uint8, device="cuda")
    qb = torch.empty_like(qa)
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    busy(torch, s1)
    ctx.eval_queries_device(pa.data_ptr(), nq, B.PRF_AES128, out.data_ptr(), s1.cuda_stream, compact=True)
    ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, B.PRF_AES128, qa.data_ptr(), qb.data_ptr(),
                           s2.cuda_stream, compact=True)
    torch.cuda.synchronize()
    assert np.array_equal(qa.cpu().numpy().reshape(nq, -1), ctx.pack_queries(ka))
    assert np.array_equal(qb.cpu().numpy().reshape(nq, -1), ctx.pack_queries(kb))
    ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_generator_leaves_cached_plan_alone(torch_cuda, kind):
    """a generator call between two cached evaluations changes neither their results nor last_launches"""
    torch = torch_cuda
    ctx, tables = make_context(kind, KINDS[kind][2], 4, 80)
    nq = 33
    alphas, seeds = random_queries(ctx, nq, 81)
    ka, _ = host_queries(ctx, alphas, seeds, B.PRF_CHACHA20)
    keys = torch.from_numpy(ctx.pack_queries(ka)).cuda()
    st = torch.cuda.current_stream()
    outs = []
    for step in range(3):
        if step == 2:
            a_dev, s_dev = torch.from_numpy(alphas).cuda(), torch.from_numpy(seeds).cuda()
            qa = torch.empty(nq * ctx.query_bytes, dtype=torch.uint8, device="cuda")
            qb = torch.empty_like(qa)
            ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, B.PRF_AES128, qa.data_ptr(), qb.data_ptr(),
                                   st.cuda_stream, compact=True)
        out = torch.full((nq, ctx.nbins, 4), -1, dtype=torch.int32, device="cuda")
        ctx.eval_queries_device(keys.data_ptr(), nq, B.PRF_CHACHA20, out.data_ptr(), st.cuda_stream, compact=True)
        torch.cuda.synchronize()
        outs.append((out.cpu().numpy(), ctx.last_launches))
    assert np.array_equal(outs[1][0], outs[2][0]) and np.array_equal(outs[0][0], outs[1][0])
    assert outs[1][1] == outs[2][1]
    ctx.close()


# ---- Python layers ----------------------------------------------------------------------------------------

def test_binned_dpf_gen_queries_device(torch_cuda):
    torch = torch_cuda
    import dpf
    sizes = KINDS["standard"][2]
    tables = [torch.from_numpy(random_table(n, 16, seed=90 + g)) for g, n in enumerate(sizes)]
    d = dpf.BinnedDPF(prf=dpf.DPF.PRF_AES128)
    d.eval_init(tables)
    nq = 5
    rng = np.random.RandomState(91)
    idx = np.stack([rng.randint(0, n, size=nq) for n in sizes], axis=1).astype(np.int64)
    seeds = rng.randint(0, 256, size=(nq, len(sizes), 44)).astype(np.uint8)
    idx_dev, seeds_dev = torch.from_numpy(idx).cuda(), torch.from_numpy(seeds).cuda()
    for compact in (True, False):
        qa, qb = d.gen_queries_device(idx_dev, seeds_dev, compact=compact)
        assert qa.is_cuda and qa.dtype == (torch.uint8 if compact else torch.int32)
        ra, rb = d.eval_queries_device(qa), d.eval_queries_device(qb)
        rec = reconstruct("standard", ra.cpu().numpy(), rb.cpu().numpy())
        assert np.array_equal(rec, selected_rows([t.numpy() for t in tables], idx))
        if not compact:
            for g, n in enumerate(sizes):
                ha, _ = B.gen_batch_secure(idx[:, g], n, seeds[:, g].tobytes(), B.PRF_AES128)
                assert np.array_equal(qa.cpu().numpy()[:, g], ha)
    qa, qb = d.gen_queries_device(idx_dev)                    # seeds from os.urandom
    rec = reconstruct("standard", d.eval_queries_device(qa).cpu().numpy(), d.eval_queries_device(qb).cpu().numpy())
    assert np.array_equal(rec, selected_rows([t.numpy() for t in tables], idx))
    for bad in (seeds_dev.cpu(), seeds_dev.int(), seeds_dev[:, :, :40], seeds_dev[:4], "seeds"):
        with pytest.raises(Exception, match=r"BinnedDPF\.gen_queries_device: seeds_dev must be a contiguous uint8 \[5, 4, 44\]"):
            d.gen_queries_device(idx_dev, bad)
    with pytest.raises(Exception, match=r"indices_dev must be a contiguous int64 \[Q, 4\] tensor on cuda:0"):
        d.gen_queries_device(idx_dev.cpu())
    d.close()


@pytest.mark.parametrize("kind", ["et", "xor"])
def test_dpf_cpp_gen_queries(torch_cuda, kind):
    """dpf_cpp.group_gen_queries_device on the contexts of group_init_et / _xor, and its refusals"""
    torch = torch_cuda
    import dpf
    cpp = dpf.dpf_cpp
    sizes = KINDS[kind][2]
    tables = [torch.from_numpy(random_table(n, 2, seed=100 + g)) for g, n in enumerate(sizes)]
    buf = getattr(cpp, "group_init_" + kind)(tables, 0)
    nq = 3
    rng = np.random.RandomState(101)
    alphas = np.stack([rng.randint(0, n, size=nq) for n in sizes], axis=1).astype(np.int64)
    seeds = rng.randint(0, 256, size=(nq, len(sizes), 44)).astype(np.uint8)
    a_dev, s_dev = torch.from_numpy(alphas).cuda(), torch.from_numpy(seeds).cuda()
    qa = torch.empty((nq, len(sizes), B.KEY_WORDS), dtype=torch.int32, device="cuda")
    qb = torch.empty_like(qa)
    st = torch.cuda.current_stream().cuda_stream
    cpp.group_gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, buf, B.PRF_SALSA20, qa.data_ptr(), qb.data_ptr(), st)
    torch.cuda.synchronize()
    for g, n in enumerate(sizes):
        ha, hb = host_gen(KINDS[kind][1], alphas[:, g], n, seeds[:, g].tobytes(), B.PRF_SALSA20)
        assert np.array_equal(qa.cpu().numpy()[:, g], ha) and np.array_equal(qb.cpu().numpy()[:, g], hb)
    for args, what in [((nq, B.PRF_SALSA20, qa.data_ptr() + 4, False), "16-byte aligned"),
                       ((0, B.PRF_SALSA20, qa.data_ptr(), False), "nqueries=0 out of range"),
                       ((nq, 4, qa.data_ptr(), True), "unknown prf id 4")]:
        with pytest.raises(RuntimeError, match=r"group_gen_queries_device: .*" + what):
            cpp.group_gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), args[0], buf, args[1], args[2], qb.data_ptr(),
                                         st, args[3])
    cpp.eval_free(buf)


def test_refusals_on_a_live_context(torch_cuda):
    """EINVAL in the order of b200dpf_group_eval_queries_device; ESTATE on a plain context; nothing written"""
    torch = torch_cuda
    ctx, _ = make_context("xor", KINDS["xor"][2], 1, 110)
    plain = B.Context(random_table(256, 1, seed=111), xor=True)
    L = B.lib()
    buf = torch.full((4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    nbins = ctx.nbins
    for args, what in [((p, p, 0, B.PRF_AES128, B.KEYS_WIRE, p, p), "nqueries=0 out of range"),
                       ((p, p, (1 << 24) // nbins + 1, B.PRF_AES128, B.KEYS_WIRE, p, p), "out of range"),
                       ((p, p, 1, 4, B.KEYS_WIRE, p, p), "unknown prf id 4"),
                       ((p, p, 1, B.PRF_AES128, 2, p, p), "unknown key_format 2"),
                       ((0, p, 1, B.PRF_AES128, B.KEYS_WIRE, p, p), "null buffer"),
                       ((p, 0, 1, B.PRF_AES128, B.KEYS_WIRE, p, p), "null buffer"),
                       ((p, p, 1, B.PRF_AES128, B.KEYS_WIRE, 0, p), "null buffer"),
                       ((p, p, 1, B.PRF_AES128, B.KEYS_COMPACT, p + 8, p), "16-byte aligned"),
                       ((p, p, 1, B.PRF_AES128, B.KEYS_COMPACT, p, p + 4), "16-byte aligned")]:
        a, s, nq, prf, fmt, oa, ob = args
        rc = L.b200dpf_group_gen_queries_device(ctx.handle, C.c_void_p(a), C.c_void_p(s), nq, prf, fmt, C.c_void_p(oa),
                                                C.c_void_p(ob), None)
        assert rc == -1 and what in L.b200dpf_last_error().decode(), what
    rc = L.b200dpf_group_gen_queries_device(plain.handle, C.c_void_p(p), C.c_void_p(p), 1, B.PRF_AES128, B.KEYS_WIRE,
                                            C.c_void_p(p), C.c_void_p(p), None)
    assert rc == -4 and "not a grouped context" in L.b200dpf_last_error().decode()
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == SENTINEL).all()
    plain.close()
    ctx.close()
