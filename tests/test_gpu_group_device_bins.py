"""Grouped (batch-PIR) evaluation from a device-resident bin list, planned on the GPU (b200dpf_group_eval_device_bins).
Every result is compared bit for bit with b200dpf_group_eval_device called with the same bins on the host, and every
pair reconstructs its row (a - b, or a ^ b, = table[bin][alpha]).  After each call the lists the device planned (the
key-group and work-unit counts, the descriptors, the work units and the order list) must equal those the host planner
made for the same bins.  Also covered: every kind and PRF, entry sizes 1 to 128, batches of 1 to 65,536 keys, bin mixes
(uniform, one bin, one key per bin, mostly empty bins, 31/32/33 keys per bin, the tiled batch-PIR shape), trimmed bins,
a forced work-item size, out-of-range bins, ordering against the other entry points and row updates over several
streams, and calls that return while their stream is still blocked."""
import os
import sys
import time

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

# per kind: GroupContext keyword, bin sizes of the mixed-size tests (the smallest each kind takes first), the size of
# the bins of the one-size tests
KINDS = {
    "standard": ({}, [2, 64, 1 << 10, 1 << 12, 1 << 14], 1 << 10),
    "et": ({"early_termination": True}, [8, 64, 1 << 10, 1 << 12, 1 << 14], 1 << 10),
    "xor": ({"xor": True}, [256, 512, 1 << 10, 1 << 12, 1 << 14], 1 << 10),
}
MIXES = ["uniform", "one_bin", "one_per_bin", "many_empty", "counts_31_32_33", "tiled"]


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


def keys_for(kind, sizes, bins, prf, seed, trimmed=False):
    """both servers' keys for the given bins (key b for a random row of bin bins[b]) and the rows they select;
    keys whose bin is out of range are keys of bin 0"""
    rng = np.random.RandomState(seed)
    nbins = len(sizes)
    home = np.where((bins >= 0) & (bins < nbins), bins, 0)
    ka = np.zeros((len(bins), B.KEY_WORDS), np.int32)
    kb = np.zeros_like(ka)
    alphas = np.zeros(len(bins), np.int64)
    for n in sorted(set(sizes[g] for g in np.unique(home))):
        sel = np.nonzero(np.array([sizes[g] for g in home]) == n)[0]
        rows = rng.randint(0, n, size=len(sel)).astype(np.int64)
        idx = np.array([B.trimmed_alpha(int(r), n, KIND_SUFFIX[kind]) for r in rows], np.int64) if trimmed else rows
        dom = B.trimmed_domain(n, KIND_SUFFIX[kind]) if trimmed else n
        a, b = gen_keys(kind, idx, dom, prf, rng)
        ka[sel], kb[sel], alphas[sel] = a, b, rows
    return ka, kb, alphas


KIND_SUFFIX = {"standard": "", "et": "_et", "xor": "_xor"}


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
    if mix == "tiled":
        return np.tile(np.arange(nbins, dtype=np.int32), 9)
    raise ValueError(mix)


def reconstruct(kind, a, b):
    if kind == "xor":
        return (a.view(np.uint32) ^ b.view(np.uint32)).view(np.int32)
    return (a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32)


def eval_bins(torch, ctx, keys, bins, prf, stream=None, bad=False):
    """eval_device_bins on keys and bins uploaded with torch; the result (and the bad-key count) back on the host"""
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys)).cuda()
    bins_dev = torch.from_numpy(np.ascontiguousarray(bins, np.int32)).cuda()
    out = torch.full((len(keys), ctx.entry_size), -1, dtype=torch.int32, device="cuda")
    bad_dev = torch.full((1,), 12345, dtype=torch.int64, device="cuda")
    st = stream if stream is not None else torch.cuda.current_stream()
    st.wait_stream(torch.cuda.current_stream())
    ctx.eval_device_bins(keys_dev.data_ptr(), bins_dev.data_ptr(), len(keys), prf, out.data_ptr(), bad_dev.data_ptr(),
                         st.cuda_stream)
    st.synchronize()
    return (out.cpu().numpy(), int(bad_dev.item())) if bad else out.cpu().numpy()


def eval_host_bins(torch, ctx, keys, bins, prf):
    """b200dpf_group_eval_device with the bins on the host: the reference of every comparison"""
    keys_dev = torch.from_numpy(np.ascontiguousarray(keys)).cuda()
    out = torch.full((len(keys), ctx.entry_size), -1, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream()
    ctx.eval_device(keys_dev.data_ptr(), bins, prf, out.data_ptr(), st.cuda_stream)
    st.synchronize()
    return out.cpu().numpy()


def check_plan_invariant(ctx, nvalid, caller=None):
    """the device lists of the last eval_device_bins call equal the host lists of the last eval_device call, which
    ran on the keys caller[0], caller[1], .. of the device call (None: on all of them, in order)"""
    dc, dd, du, do = ctx.plan_lists(True)
    hc, hd, hu, ho = ctx.plan_lists(False)
    assert dc[0] == hc[0] and dc[1] == hc[1], (dc, hc)
    assert np.array_equal(dd, hd)
    assert np.array_equal(du, hu)
    ho = ho[:nvalid].copy()
    if caller is not None:
        ho[:, 0] = caller[ho[:, 0]]
    assert np.array_equal(do[:nvalid], ho)
    return dc


def check_batch(torch, kind, ctx, tables, bins, prf, seed, trimmed=False):
    sizes = [t.shape[0] for t in tables]
    ka, kb, alphas = keys_for(kind, sizes, bins, prf, seed, trimmed)
    ra, bad = eval_bins(torch, ctx, ka, bins, prf, bad=True)
    assert bad == 0
    assert ctx.last_launches == (ctx.entry_size + 15) // 16      # the evaluation launches, timed alone
    assert ctx.last_device_ms > 0
    want = eval_host_bins(torch, ctx, ka, bins, prf)
    assert np.array_equal(ra, want)
    check_plan_invariant(ctx, len(bins))
    rb = eval_bins(torch, ctx, kb, bins, prf)
    assert np.array_equal(rb, eval_host_bins(torch, ctx, kb, bins, prf))
    rows = np.stack([tables[g][a] for g, a in zip(bins, alphas)])
    assert np.array_equal(reconstruct(kind, ra, rb), rows)


@pytest.mark.parametrize("mix", MIXES)
@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("kind", list(KINDS))
def test_mixes_bit_exact(torch_cuda, kind, prf, mix):
    kw, _, n = KINDS[kind]
    nbins = 40
    rng = np.random.RandomState(100 * MIXES.index(mix) + 10 * prf + list(KINDS).index(kind))
    bins = make_bins(mix, nbins, rng)
    tables = [random_table(n, 16, seed=7 * g + prf) for g in range(nbins)]
    ctx = B.GroupContext(tables, **kw)
    try:
        check_batch(torch_cuda, kind, ctx, tables, bins, prf, seed=11 + prf)
    finally:
        ctx.close()


@pytest.mark.parametrize("e", [1, 16, 40, 128])
@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("kind", list(KINDS))
def test_mixed_sizes_entry_sizes(torch_cuda, kind, prf, e):
    kw, sizes, _ = KINDS[kind]
    sizes = sizes * 3                      # 15 bins of five sizes
    rng = np.random.RandomState(e + 10 * prf)
    bins = rng.randint(0, len(sizes), size=500).astype(np.int32)
    tables = [random_table(n, e, seed=100 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **kw)
    try:
        check_batch(torch_cuda, kind, ctx, tables, bins, prf, seed=20 + e)
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_batch_sizes(torch_cuda, kind):
    """1 to 65,536 (bin, key) pairs on one context: the host half of the plan is made again for every new nkeys, and
    the scratch grows"""
    kw, _, n = KINDS[kind]
    nbins = 256
    tables = [random_table(n, 16, seed=300 + g) for g in range(nbins)]
    ctx = B.GroupContext(tables, **kw)
    rng = np.random.RandomState(5)
    try:
        for nkeys, prf in ((1, B.PRF_AES128), (2, B.PRF_CHACHA20), (31, B.PRF_AES128), (33, B.PRF_SALSA20),
                           (4097, B.PRF_CHACHA20), (65536, B.PRF_AES128), (100, B.PRF_DUMMY)):
            bins = rng.randint(0, nbins, size=nkeys).astype(np.int32)
            check_batch(torch_cuda, kind, ctx, tables, bins, prf, seed=nkeys)
        bins = np.tile(np.arange(nbins, dtype=np.int32), 256)          # the tiled batch-PIR shape, 65,536 pairs
        check_batch(torch_cuda, kind, ctx, tables, bins, B.PRF_CHACHA20, seed=77)
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_trimmed_bins_and_forced_subtree(torch_cuda, kind):
    kw, sizes, _ = KINDS[kind]
    trimmed_sizes = [1, 3, 100, 700, 3001, 5000, sizes[-1] - 1]
    tables = [random_table(n, 24, seed=400 + g) for g, n in enumerate(trimmed_sizes)]
    ctx = B.GroupContext(tables, trimmed=True, **{k: v for k, v in kw.items()})
    rng = np.random.RandomState(9)
    try:
        for prf in PRFS:
            bins = rng.randint(0, len(trimmed_sizes), size=600).astype(np.int32)
            check_batch(torch_cuda, kind, ctx, tables, bins, prf, seed=prf, trimmed=True)
        bins = rng.randint(0, len(trimmed_sizes), size=400).astype(np.int32)
        for s in (1, 2, 3, 7):                 # the work-item size is a tuning knob only
            ctx.set_subtree_log2(s)
            check_batch(torch_cuda, kind, ctx, tables, bins, B.PRF_CHACHA20, seed=50 + s, trimmed=True)
        ctx.set_subtree_log2(0)
        check_batch(torch_cuda, kind, ctx, tables, bins, B.PRF_CHACHA20, seed=60, trimmed=True)
    finally:
        ctx.close()


def do_tail(ctx, nvalid):
    """the caller's indices at the sorted positions past the valid keys of the last eval_device_bins call"""
    return ctx.plan_lists(True)[3][nvalid:, 0].tolist()


@pytest.mark.parametrize("prf", [B.PRF_CHACHA20, B.PRF_AES128])
@pytest.mark.parametrize("kind", list(KINDS))
def test_out_of_range_bins(torch_cuda, kind, prf):
    kw, sizes, _ = KINDS[kind]
    nbins = len(sizes)
    tables = [random_table(n, 40, seed=500 + g) for g, n in enumerate(sizes)]
    ctx = B.GroupContext(tables, **kw)
    rng = np.random.RandomState(prf)
    try:
        for nbad in (1, 37, 200):
            bins = rng.randint(0, nbins, size=400).astype(np.int32)
            bad_at = rng.choice(len(bins), size=nbad, replace=False)
            bins[bad_at] = rng.choice([-1, -7, -2**31, nbins, nbins + 5, 2**31 - 1], size=nbad)
            ka, kb, alphas = keys_for(kind, sizes, bins, prf, seed=nbad)
            good = np.setdiff1d(np.arange(len(bins)), bad_at)
            ra, bad = eval_bins(torch_cuda, ctx, ka, bins, prf, bad=True)
            assert bad == nbad
            assert not ra[bad_at].any()
            assert np.array_equal(ra[good], eval_host_bins(torch_cuda, ctx, ka[good], bins[good], prf))
            counts = check_plan_invariant(ctx, len(good), caller=good)
            assert set(do_tail(ctx, len(good))) == set(bad_at)       # the out-of-range keys form the tail
            assert counts[3] == nbad
            rb = eval_bins(torch_cuda, ctx, kb, bins, prf)
            rows = np.stack([tables[bins[i]][alphas[i]] for i in good])
            assert np.array_equal(reconstruct(kind, ra[good], rb[good]), rows)
        every = np.full(50, -3, np.int32)          # no key has a bin: no key group at all
        ka, _, _ = keys_for(kind, sizes, every, prf, seed=1)
        ra, bad = eval_bins(torch_cuda, ctx, ka, every, prf, bad=True)
        assert bad == 50 and not ra.any()
    finally:
        ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_ordering_over_streams(torch_cuda, kind):
    """calls on one context interleaved with every other grouped entry point and row updates, spread over three
    streams with no host synchronisation, give the results of running them one at a time; the cached query plan
    still holds afterwards"""
    torch = torch_cuda
    kw, _, n = KINDS[kind]
    nbins, prf = 16, B.PRF_AES128
    tables = [random_table(n, 16, seed=600 + g) for g in range(nbins)]
    rng = np.random.RandomState(3)
    q = 6
    tiled = np.tile(np.arange(nbins, dtype=np.int32), q)
    qa, _, _ = keys_for(kind, [n] * nbins, tiled, prf, seed=1)
    batches = []
    for i in range(4):
        bins = rng.randint(0, nbins, size=300 + 50 * i).astype(np.int32)
        batches.append((keys_for(kind, [n] * nbins, bins, prf, seed=10 + i)[0], bins))
    upd_bins = rng.randint(0, nbins, size=20).astype(np.int32)
    upd_idx = rng.randint(0, n, size=20).astype(np.int64)
    upd_rows = rng.randint(-2**31, 2**31, size=(20, 16)).astype(np.int32)

    def run(ctx, streams, sync):
        """the sequence on `ctx`; `sync`: each step finishes before the next starts"""
        outs = []

        def dev(t):
            return torch.from_numpy(np.ascontiguousarray(t)).cuda()
        ins = [(dev(k), dev(b)) for k, b in batches]
        q_dev = dev(qa)
        torch.cuda.synchronize()
        steps = []
        for i, (k, b) in enumerate(ins):
            steps.append(("bins", i))
            steps.append(("device", i))
            if i == 1:
                steps.append(("update", None))
            if i == 2:
                steps.append(("host", i))
            steps.append(("queries", None))
        for j, (what, i) in enumerate(steps):
            st = streams[j % len(streams)]
            if what == "bins":
                k, b = ins[i]
                out = torch.empty((len(batches[i][1]), 16), dtype=torch.int32, device="cuda")
                ctx.eval_device_bins(k.data_ptr(), b.data_ptr(), len(batches[i][1]), prf, out.data_ptr(), 0, st.cuda_stream)
                outs.append(out)
            elif what == "device":
                k, _ = ins[i]
                out = torch.empty((len(batches[i][1]), 16), dtype=torch.int32, device="cuda")
                ctx.eval_device(k.data_ptr(), batches[i][1], prf, out.data_ptr(), st.cuda_stream)
                outs.append(out)
            elif what == "queries":
                out = torch.empty((q, nbins, 16), dtype=torch.int32, device="cuda")
                ctx.eval_queries_device(q_dev.data_ptr(), q, prf, out.data_ptr(), st.cuda_stream)
                outs.append(out)
            elif what == "host":
                outs.append(torch.from_numpy(ctx.eval(batches[i][0], batches[i][1], prf)))
            else:
                ctx.update_rows(upd_bins, upd_idx, upd_rows)
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return [o.cpu().numpy() for o in outs]

    ref_ctx = B.GroupContext(tables, **kw)
    ctx = B.GroupContext(tables, **kw)
    try:
        want = run(ref_ctx, [torch.cuda.current_stream()], True)
        streams = [torch.cuda.Stream() for _ in range(3)]
        got = run(ctx, streams, False)
        assert len(got) == len(want)
        for j, (g, w) in enumerate(zip(got, want)):
            assert np.array_equal(g, w), j
        # the cached query plan is still that of q queries: a further call matches the host path on the updated table
        out = torch.empty((q, nbins, 16), dtype=torch.int32, device="cuda")
        ctx.eval_queries_device(torch.from_numpy(qa).cuda().data_ptr(), q, prf, out.data_ptr(), streams[1].cuda_stream)
        streams[1].synchronize()
        assert np.array_equal(out.cpu().numpy().reshape(-1, 16), ctx.eval(qa, tiled, prf))
    finally:
        ctx.close()
        ref_ctx.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_no_host_wait(torch_cuda, kind):
    """with its stream held behind a 2^30-cycle sleep on another stream, a call returns long before the sleep ends,
    and so does a second call queued behind the first; both are right after synchronising"""
    torch = torch_cuda
    kw, _, n = KINDS[kind]
    nbins, prf = 64, B.PRF_CHACHA20
    tables = [random_table(n, 16, seed=700 + g) for g in range(nbins)]
    rng = np.random.RandomState(4)
    bins = rng.randint(0, nbins, size=5000).astype(np.int32)
    ka, kb, alphas = keys_for(kind, [n] * nbins, bins, prf, seed=2)
    ctx = B.GroupContext(tables, **kw)
    try:
        want_a = eval_host_bins(torch, ctx, ka, bins, prf)
        want_b = eval_host_bins(torch, ctx, kb, bins, prf)
        ka_dev, kb_dev = torch.from_numpy(ka).cuda(), torch.from_numpy(kb).cuda()
        bins_dev = torch.from_numpy(bins).cuda()
        out_a = torch.empty((len(bins), 16), dtype=torch.int32, device="cuda")
        out_b = torch.empty_like(out_a)
        sleeper, st = torch.cuda.Stream(), torch.cuda.Stream()
        # warm-up on the same stream and nkeys: the plan, the scratch and the kernels' attributes are ready
        ctx.eval_device_bins(ka_dev.data_ptr(), bins_dev.data_ptr(), len(bins), prf, out_a.data_ptr(), 0, st.cuda_stream)
        torch.cuda.synchronize()
        out_a.fill_(-1)
        out_b.fill_(-1)
        torch.cuda.synchronize()
        with torch.cuda.stream(sleeper):
            t0 = time.perf_counter()
            torch.cuda._sleep(1 << 30)         # about 0.5 s at 2 GHz
            ev = torch.cuda.Event()
            ev.record(sleeper)
        st.wait_event(ev)
        t1 = time.perf_counter()
        ctx.eval_device_bins(ka_dev.data_ptr(), bins_dev.data_ptr(), len(bins), prf, out_a.data_ptr(), 0, st.cuda_stream)
        t2 = time.perf_counter()
        ctx.eval_device_bins(kb_dev.data_ptr(), bins_dev.data_ptr(), len(bins), prf, out_b.data_ptr(), 0, st.cuda_stream)
        t3 = time.perf_counter()
        still_sleeping = not ev.query()
        torch.cuda.synchronize()
        t4 = time.perf_counter()
        assert still_sleeping, "the sleep ended before both calls returned"
        assert t3 - t1 < 0.25 * (t4 - t0), (t2 - t1, t3 - t2, t4 - t0)
        assert np.array_equal(out_a.cpu().numpy(), want_a)
        assert np.array_equal(out_b.cpu().numpy(), want_b)
        rows = np.stack([tables[g][a] for g, a in zip(bins, alphas)])
        assert np.array_equal(reconstruct(kind, want_a, want_b), rows)
    finally:
        ctx.close()


def test_python_surfaces(torch_cuda):
    """dpf_cpp.group_eval_device_bins and BinnedDPF.eval_gpu_device_bins give what eval_gpu_device gives"""
    torch = torch_cuda
    import dpf
    d = dpf.BinnedDPF(prf=dpf.DPF.PRF_AES128)
    sizes = [1 << 8, 1 << 10, 1 << 12]
    tables = [torch.from_numpy(random_table(n, 20, seed=800 + g)) for g, n in enumerate(sizes)]
    d.eval_init(tables)
    rng = np.random.RandomState(8)
    bins = rng.randint(0, 3, size=90).astype(np.int32)
    alphas = [int(rng.randint(0, sizes[g])) for g in bins]
    pairs = [d.gen_in_bin(int(g), a) for g, a in zip(bins, alphas)]
    ka = torch.stack([p[0] for p in pairs]).cuda()
    kb = torch.stack([p[1] for p in pairs]).cuda()
    bins_dev = torch.from_numpy(bins).cuda()
    bad = torch.full((1,), 99, dtype=torch.int64, device="cuda")
    ra = d.eval_gpu_device_bins(ka, bins_dev, bad_dev=bad)
    rb = torch.empty_like(ra)
    d.eval_gpu_device_bins(kb, bins_dev, out_dev=rb)
    torch.cuda.synchronize()
    assert int(bad.item()) == 0
    assert torch.equal(ra, d.eval_gpu_device(ka, bins))
    assert torch.equal(rb, d.eval_gpu_device(kb, bins))
    diff = (ra.cpu().numpy().astype(np.uint32) - rb.cpu().numpy().astype(np.uint32)).astype(np.int32)
    assert np.array_equal(diff, np.stack([tables[g][a].numpy() for g, a in zip(bins, alphas)]))
    out = torch.empty_like(ra)
    dpf.dpf_cpp.group_eval_device_bins(ka.data_ptr(), bins_dev.data_ptr(), len(bins), d.buffers, d.prf_method,
                                       out.data_ptr(), 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(out, ra)
