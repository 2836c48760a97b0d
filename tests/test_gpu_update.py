"""Row updates of a live table (b200dpf_update_rows*, DPF.update_rows, BinnedDPF.update_rows,
ShardedDPF.update_rows): results after an update equal the oracle on a numpy copy of the table with the
same updates applied in order, and evaluations are ordered against updates on every stream."""
import os
import socket
import sys

import numpy as np
import pytest

import b200dpf
from common import oracle_dot_mt, random_table, seeded_keys

pytestmark = pytest.mark.gpu

ALL_PRFS = [0, 1, 2, 3]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


def apply_updates(table, idx, rows):
    """The expected table: updates applied one after the other, so the last occurrence wins."""
    new = table.copy()
    for i, r in zip(idx, rows):
        new[i] = r
    return new


def update_list(n, e, seed, count=12):
    """Indices with 0, n-1 and repeats carrying distinct rows (last-wins is observable), plus random rows."""
    rng = np.random.RandomState(seed)
    picks = rng.randint(0, n, size=count)
    idx = np.concatenate([[0, n - 1], picks, picks[:3], [0]]).astype(np.int64)
    rows = rng.randint(-2**31, 2**31, size=(len(idx), e), dtype=np.int64).astype(np.int32)
    return idx, rows


def reconstruct(a, b):
    return (a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32)


def keys_at(alphas, n, prf, seed):
    alphas = np.asarray(alphas, np.int64)
    return b200dpf.gen_batch(alphas, n, np.arange(len(alphas)) + seed, prf)


@pytest.mark.parametrize("prf", ALL_PRFS)
@pytest.mark.parametrize("n,e", [(128, 1), (1 << 14, 5), (1 << 14, 16), (1 << 14, 40), (1 << 16, 200), (1 << 20, 16)])
def test_single_context(oracle, torch_cuda, prf, n, e):
    table = random_table(n, e, seed=n + e + prf)
    idx, rows = update_list(n, e, seed=n * 3 + e + prf)
    new = apply_updates(table, idx, rows)
    ctx = b200dpf.Context(table)
    ctx.update_rows(idx, rows)
    nchk = 2 if n >= (1 << 20) else 6
    rng = np.random.RandomState(prf)
    for batch in (1, 7, 512):
        # every updated index is queried (when the batch is large enough), the rest at random
        alphas = np.concatenate([np.unique(idx), rng.randint(0, n, size=batch)])[:batch]
        ka, kb = keys_at(alphas, n, prf, seed=batch)
        a, b = ctx.eval(ka, prf), ctx.eval(kb, prf)
        assert np.array_equal(reconstruct(a, b), new[alphas]), (n, e, batch)
        assert np.array_equal(a[:nchk], oracle_dot_mt(oracle, ka[:nchk], prf, new)), (n, e, batch)
    if prf != 3 and (n, e) == (1 << 14, 16):
        ctx.set_option("tma_rows", 1)
        ctx.update_rows(idx[::-1].copy(), rows[::-1].copy())        # reversed: the first rows win now
        new = apply_updates(new, idx[::-1], rows[::-1])
        alphas = np.concatenate([np.unique(idx), rng.randint(0, n, size=512)])[:512]
        ka, kb = keys_at(alphas, n, prf, seed=3)
        a, b = ctx.eval(ka, prf), ctx.eval(kb, prf)
        assert np.array_equal(reconstruct(a, b), new[alphas])
        assert np.array_equal(a[:nchk], oracle.eval_dot(ka[:nchk], prf, new))
    ctx.close()


@pytest.mark.parametrize("shards", [2, 4, 8])
def test_entry_range_shards(oracle, torch_cuda, shards):
    """Every shard takes the same full list, host or device path; the partials equal the per-shard oracle on
    the updated table and add up to the whole."""
    torch = torch_cuda
    n, e, prf, batch = 1 << 14, 16, 3, 40
    table = random_table(n, e, seed=shards)
    idx, rows = update_list(n, e, seed=shards + 100, count=200)
    new = apply_updates(table, idx, rows)
    ka, _, _ = seeded_keys(b200dpf.gen, n, batch, prf, seed=shards)
    idx_dev, rows_dev = torch.from_numpy(idx).cuda(), torch.from_numpy(rows).cuda()
    total = np.zeros((batch, e), np.uint32)
    for r in range(shards):
        parts = []
        for path in ("host", "device"):
            ctx = b200dpf.Context(table, shard_rank=r, shard_count=shards)
            if path == "host":
                ctx.update_rows(idx, rows)
            else:
                ctx.update_rows_device(idx_dev.data_ptr(), rows_dev.data_ptr(), len(idx))
                torch.cuda.synchronize()
            parts.append(ctx.eval(ka, prf))
            ctx.close()
        assert np.array_equal(parts[0], parts[1]), r
        for b in range(3):
            assert np.array_equal(parts[0][b], oracle.eval_dot_shard(ka[b], prf, new, r * n // shards, n // shards)), (r, b)
        total += parts[0].astype(np.uint32)
    assert np.array_equal(total.astype(np.int32), oracle.eval_dot(ka, prf, new))


def test_ordering_device_path(torch_cuda):
    """eval A on S1, update on S2, eval B on S1, nothing synchronised in between: A sees only the old
    table, B only the new one.  Then the same with the host path between two unsynchronised evaluations."""
    torch = torch_cuda
    n, e, prf, batch = 1 << 20, 16, 3, 512
    table = random_table(n, e, seed=41)
    ka, _, _ = seeded_keys(b200dpf.gen, n, batch, prf, seed=42)
    rng = np.random.RandomState(43)
    idx = rng.randint(0, n, size=1024).astype(np.int64)
    rows = rng.randint(-2**31, 2**31, size=(1024, e), dtype=np.int64).astype(np.int32)
    new = apply_updates(table, idx, rows)
    want_old = b200dpf.Context(table).eval(ka, prf)
    ref_new = b200dpf.Context(new)
    want_new = ref_new.eval(ka, prf)
    ref_new.close()
    assert not np.array_equal(want_old, want_new)

    ctx = b200dpf.Context(table)
    keys = torch.from_numpy(ka).cuda()
    idx_dev, rows_dev = torch.from_numpy(idx).cuda(), torch.from_numpy(rows).cuda()
    out_a = torch.empty((batch, e), dtype=torch.int32, device="cuda")
    out_b = torch.empty_like(out_a)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    ctx.eval_device(keys.data_ptr(), batch, prf, out_a.data_ptr(), s1.cuda_stream)
    ctx.update_rows_device(idx_dev.data_ptr(), rows_dev.data_ptr(), len(idx), s2.cuda_stream)
    ctx.eval_device(keys.data_ptr(), batch, prf, out_b.data_ptr(), s1.cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(out_a.cpu().numpy(), want_old)
    assert np.array_equal(out_b.cpu().numpy(), want_new)
    ctx.close()

    ctx = b200dpf.Context(table)
    torch.cuda.synchronize()
    ctx.eval_device(keys.data_ptr(), batch, prf, out_a.data_ptr(), s1.cuda_stream)
    ctx.update_rows(idx, rows)
    ctx.eval_device(keys.data_ptr(), batch, prf, out_b.data_ptr(), s1.cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(out_a.cpu().numpy(), want_old)
    assert np.array_equal(out_b.cpu().numpy(), want_new)
    ctx.close()


def test_bad_input(oracle, torch_cuda):
    import ctypes as C
    torch = torch_cuda
    L = b200dpf.lib()
    n, e, prf = 4096, 16, 2
    table = random_table(n, e, seed=51)
    ka, kb, alphas = seeded_keys(b200dpf.gen, n, 20, prf, seed=52)
    ctx = b200dpf.Context(table)
    before = ctx.eval(ka, prf)
    one = np.zeros((2, e), np.int32)
    assert L.b200dpf_update_rows(ctx.handle, np.array([5, n], np.int64), one, 2) == -1
    assert b"out of range" in L.b200dpf_last_error()
    assert L.b200dpf_update_rows(ctx.handle, np.array([5, -1], np.int64), one, 2) == -1
    assert L.b200dpf_update_rows(ctx.handle, np.array([5, 6], np.int64), one, -1) == -1
    assert L.b200dpf_group_update_rows(ctx.handle, np.zeros(2, np.int32), np.array([5, 6], np.int64), one, 2) == -4
    assert np.array_equal(ctx.eval(ka, prf), before)        # nothing was applied
    with pytest.raises(b200dpf.B200DPFError, match="out of range"):
        ctx.update_rows(np.array([alphas[0], n + 3]), one)
    assert np.array_equal(ctx.eval(ka, prf), before)

    # device path: out-of-range entries are skipped, the valid ones applied, every other row unchanged
    good = np.array([alphas[0], alphas[1], 17], np.int64)
    idx = np.array([good[0], n, good[1], -1, good[2], 1 << 40], np.int64)
    rows = np.random.RandomState(53).randint(-2**31, 2**31, size=(len(idx), e), dtype=np.int64).astype(np.int32)
    new = table.copy()
    for i, r in zip(idx, rows):
        if 0 <= i < n:
            new[i] = r
    idx_dev, rows_dev = torch.from_numpy(idx).cuda(), torch.from_numpy(rows).cuda()
    ctx.update_rows_device(idx_dev.data_ptr(), rows_dev.data_ptr(), len(idx))
    torch.cuda.synchronize()
    probe = np.unique(np.concatenate([good, good - 1, good + 1, [0, n - 1]]) % n)
    pa, pb = keys_at(probe, n, prf, seed=54)
    assert np.array_equal(reconstruct(ctx.eval(pa, prf), ctx.eval(pb, prf)), new[probe])
    assert np.array_equal(ctx.eval(ka[:4], prf), oracle.eval_dot(ka[:4], prf, new))
    ctx.close()


def test_grouped_context(oracle, torch_cuda):
    sizes = [2, 128, 4096, 1 << 14]
    prf = 3
    rng = np.random.RandomState(61)
    for e in (5, 16, 40):
        tables = [random_table(n, e, seed=n + e + g) for g, n in enumerate(sizes)]
        ctx = b200dpf.GroupContext(tables)
        bins = rng.randint(0, len(sizes), size=60).astype(np.int32)
        idx = np.array([rng.randint(0, sizes[g]) for g in bins], np.int64)
        bins = np.concatenate([bins, bins[:5], [3, 3]]).astype(np.int32)            # repeats with new rows
        idx = np.concatenate([idx, idx[:5], [sizes[3] - 1, sizes[3] - 1]]).astype(np.int64)
        rows = rng.randint(-2**31, 2**31, size=(len(idx), e), dtype=np.int64).astype(np.int32)
        new = [t.copy() for t in tables]
        for g, i, r in zip(bins, idx, rows):
            new[g][i] = r
        ctx.update_rows(bins, idx, rows)
        qbins = np.concatenate([bins, rng.randint(0, len(sizes), size=30)]).astype(np.int32)
        qidx = np.concatenate([idx, [rng.randint(0, sizes[g]) for g in qbins[len(bins):]]]).astype(np.int64)
        ka, kb = [], []
        for q, (g, i) in enumerate(zip(qbins, qidx)):
            a, b = b200dpf.gen(int(i), sizes[g], 7000 + q, prf)
            ka.append(a); kb.append(b)
        ka, kb = np.stack(ka), np.stack(kb)
        a, b = ctx.eval(ka, qbins, prf), ctx.eval(kb, qbins, prf)
        assert np.array_equal(reconstruct(a, b), np.stack([new[g][i] for g, i in zip(qbins, qidx)])), e
        for g in range(len(sizes)):
            sel = np.nonzero(qbins == g)[0][:4]
            if len(sel):
                assert np.array_equal(a[sel], oracle.eval_dot(ka[sel], prf, new[g])), (e, g)
        before = ctx.eval(ka, qbins, prf)
        with pytest.raises(b200dpf.B200DPFError, match="bin 4 out of range"):
            ctx.update_rows([0, 4], [0, 0], np.zeros((2, e), np.int32))
        with pytest.raises(b200dpf.B200DPFError, match="out of range"):
            ctx.update_rows([1, 0], [5, 2], np.zeros((2, e), np.int32))              # index 2 >= n[0] = 2
        with pytest.raises(b200dpf.B200DPFError, match="b200dpf_group_update_rows"):
            b200dpf.Context.update_rows(ctx, [0], np.zeros((1, e), np.int32))
        assert np.array_equal(ctx.eval(ka, qbins, prf), before)
        ctx.close()


def test_multi_context_with_one_device(oracle, torch_cuda):
    n, e, prf = 4096, 16, 1
    table = random_table(n, e, seed=71)
    idx, rows = update_list(n, e, seed=72, count=40)
    new = apply_updates(table, idx, rows)
    ka, kb, alphas = seeded_keys(b200dpf.gen, n, 40, prf, seed=73)
    idx_dev, rows_dev = torch_cuda.from_numpy(idx).cuda(), torch_cuda.from_numpy(rows).cuda()
    for axis in (1, 2):
        ctx = b200dpf.Context.multi(table, [0], axis)
        ctx.update_rows(idx, rows)
        a, b = ctx.eval(ka, prf), ctx.eval(kb, prf)
        assert np.array_equal(a, oracle.eval_dot(ka, prf, new)), axis
        assert np.array_equal(reconstruct(a, b), new[alphas])
        with pytest.raises(b200dpf.B200DPFError, match=r"\(-1\): multi-device contexts take host buffers"):
            ctx.update_rows_device(idx_dev.data_ptr(), rows_dev.data_ptr(), len(idx))
        ctx.close()


def test_python_api(oracle, torch_cuda):
    torch = torch_cuda
    import dpf
    n, e = 1 << 12, 6
    caller = torch.from_numpy(random_table(n, e, seed=81))
    kept = caller.clone()
    d = dpf.DPF(prf=dpf.DPF.PRF_SALSA20)
    d.eval_init(caller)
    picks = [0, 5, n - 1, 5]
    rows = torch.from_numpy(np.random.RandomState(82).randint(-2**31, 2**31, size=(4, e), dtype=np.int64).astype(np.int32))
    d.update_rows(torch.tensor(picks), rows)                                 # CPU: host path
    want = kept.clone()
    for i, r in zip(picks, rows):
        want[i] = r
    assert torch.equal(caller, kept)                                          # the caller's tensor is not written
    assert torch.equal(d.table, want)
    rows2 = rows.double() * 0 + torch.arange(e, dtype=torch.float64) - 3.0   # any dtype, cast like eval_init
    idx2 = torch.tensor([7, n - 2, 7, 1]).cuda()
    d.update_rows(idx2, rows2.cuda())                                         # CUDA: device path on the current stream
    for i, r in zip(idx2.tolist(), rows2):
        want[i] = r.to(torch.int32)
    assert torch.equal(d.table, want)
    ks = [d.gen(i, n) for i in (0, 5, 7, n - 1, n - 2, 100)]
    a = d.eval_gpu([k[0] for k in ks])
    b = d.eval_gpu([k[1] for k in ks])
    assert torch.equal(a - b, want[[0, 5, 7, n - 1, n - 2, 100]])
    assert torch.equal(d.eval_cpu([k[0] for k in ks]), a)                     # eval_cpu follows the updates
    assert np.array_equal(a.numpy()[:2], oracle.eval_dot(torch.stack([ks[0][0], ks[1][0]]).numpy(), 1, want.numpy()))
    with pytest.raises(Exception, match="out of range"):
        d.update_rows(torch.tensor([n]), rows[:1])
    with pytest.raises(Exception, match="rows must be"):
        d.update_rows(torch.tensor([1]), rows[:1, :3])
    d.close()

    # allow_non_pow2: the zero padding beyond the caller's rows cannot be updated
    d = dpf.DPF(prf=dpf.DPF.PRF_CHACHA20, allow_non_pow2=True)
    t = torch.from_numpy(random_table(1000, 3, seed=83))
    d.eval_init(t)
    with pytest.raises(Exception, match=r"out of range \[0, 1000\)"):
        d.update_rows([1000], torch.ones((1, 3), dtype=torch.int32))
    d.update_rows([999], torch.full((1, 3), 9, dtype=torch.int32))
    k1, k2 = d.gen(999, 1000)
    assert torch.equal((d.eval_gpu([k1]) - d.eval_gpu([k2]))[0], torch.full((3,), 9, dtype=torch.int32))
    d.close()

    # BinnedDPF
    sizes = [256, 1024]
    tables = [torch.from_numpy(random_table(m, 16, seed=m)) for m in sizes]
    bd = dpf.BinnedDPF(prf=dpf.DPF.PRF_CHACHA20)
    bd.eval_init(tables)
    newrows = torch.arange(3 * 16, dtype=torch.int32).reshape(3, 16)
    bd.update_rows([1, 0, 1], [1023, 7, 1023], newrows)
    want_bins = [t.clone() for t in tables]
    want_bins[1][1023] = newrows[2]
    want_bins[0][7] = newrows[1]
    picks = [(1, 1023), (0, 7), (0, 8), (1, 0)]
    ks = [bd.gen_in_bin(g, i) for g, i in picks]
    qb = [g for g, _ in picks]
    a = bd.eval_gpu([k[0] for k in ks], qb)
    b = bd.eval_gpu([k[1] for k in ks], qb)
    assert torch.equal(a - b, torch.stack([want_bins[g][i] for g, i in picks]))
    for q, (g, _) in enumerate(picks):
        assert np.array_equal(a[q:q + 1].numpy(), oracle.eval_dot(ks[q][0].numpy(), 2, want_bins[g].numpy()))
    bd.close()


# ---- several GPUs (skipped on a one-GPU machine) --------------------------------------------------------

def _devices():
    import torch
    n = torch.cuda.device_count()
    return list(range(1 << (n.bit_length() - 1))) if n else []


def test_multi_device_context(oracle, torch_cuda):
    devs = _devices()
    if len(devs) < 2:
        pytest.skip("needs >= 2 GPUs")
    for n, e, prf in ((1 << 14, 16, 3), (1 << 16, 40, 2)):
        table = random_table(n, e, seed=n + e)
        idx, rows = update_list(n, e, seed=n, count=300)
        new = apply_updates(table, idx, rows)
        ka, kb, alphas = seeded_keys(b200dpf.gen, n, 70, prf, seed=e)
        want = oracle_dot_mt(oracle, ka[:8], prf, new)
        for axis in (1, 2):
            ctx = b200dpf.Context.multi(table, devs, axis)
            ctx.update_rows(idx, rows)
            a, b = ctx.eval(ka, prf), ctx.eval(kb, prf)
            assert np.array_equal(a[:8], want), (n, axis)
            assert np.array_equal(reconstruct(a, b), new[alphas])
            ctx.close()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, ret):
    for sub in ("gpu-dpf_b200", "oracle", "tests"):
        sys.path.insert(0, os.path.join(ROOT, sub))
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import b200dpf as B
    import oracle as O
    from common import random_table, seeded_keys
    from sharded import ShardedDPF
    orc = O.Oracle()
    n, e, prf = 1 << 14, 16, 3
    table = random_table(n, e, seed=91)
    rng = np.random.RandomState(92)
    idx = np.concatenate([[0, n - 1], rng.randint(0, n, size=100), [0]]).astype(np.int64)
    rows = rng.randint(-2**31, 2**31, size=(len(idx), e), dtype=np.int64).astype(np.int32)
    new = table.copy()
    for i, r in zip(idx, rows):
        new[i] = r
    ka, kb, alphas = seeded_keys(B.gen, n, 70, prf, seed=93)
    for axis in ("entries", "keys"):
        d = ShardedDPF(prf=prf, axis=axis)
        d.eval_init(torch.from_numpy(table))
        d.update_rows(torch.from_numpy(idx), torch.from_numpy(rows))
        a, b = d.eval_gpu(torch.from_numpy(ka)), d.eval_gpu(torch.from_numpy(kb))
        if rank == 0:
            assert np.array_equal(a.numpy()[:8], orc.eval_dot(ka[:8], prf, new)), axis
            rec = (a.numpy().astype(np.uint32) - b.numpy().astype(np.uint32)).astype(np.int32)
            assert np.array_equal(rec, new[alphas]), axis
        d.close()
    if rank == 0:
        ret.put("ok")
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_update_rows_nccl(torch_cuda):
    import torch.multiprocessing as mp
    world = torch_cuda.cuda.device_count()
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 1 << (world.bit_length() - 1)
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, ret)) for r in range(world)]
    [p.start() for p in procs]
    [p.join(300) for p in procs]
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert ret.get(timeout=5) == "ok"
