"""Early-terminated keys (four table rows per GGM leaf) on the GPU: every evaluation path of a
b200dpf_create_et context, bit-exact against the per-index oracle (tests/et_oracle.py) at small n
and against the host evaluation (itself checked against the oracle in test_et_host.py) at large n."""
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
import et_oracle  # noqa: E402
import oracle  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
EINVAL = -1


@pytest.fixture(scope="module")
def orc():
    return oracle.Oracle()


def keys_for(n, batch, prf, seed=0):
    rng = np.random.RandomState(seed + 17 * prf + n % 1000003)
    alphas = rng.randint(0, n, size=batch).astype(np.int64)
    alphas[: min(batch, 4)] = [0, n - 1, 1, 2][: min(batch, 4)]
    seeds = rng.randint(0, 256, size=44 * batch).astype(np.uint8).tobytes()
    a, b = B.gen_batch_et(alphas, n, seeds, prf)
    return a, b, alphas


def host_dot(keys, prf, table):
    return et_oracle.dot_u32(np.stack([B.eval_cpu_et(k, prf) for k in keys]), table)


def reconstructs(ra, rb, table, alphas):
    return np.array_equal((ra.view(np.uint32) - rb.view(np.uint32)).view(np.int32), table[alphas])


GRID = [  # (n, E, B): a thinned grid over n, entry sizes around the 16 / 32 / 64-column passes, batch sizes
    (8, 1, 1), (8, 17, 3), (128, 5, 31), (128, 33, 32), (1024, 16, 33), (1024, 200, 3),
    (1024, 32, 512), (1 << 14, 16, 512), (1 << 14, 128, 33), (1 << 14, 17, 1), (1 << 16, 16, 31), (1 << 16, 33, 17),
]


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("n,e,batch", GRID)
def test_bit_exact_vs_oracle(prf, n, e, batch, orc):
    table = random_table(n, e, seed=n + e)
    a, b, alphas = keys_for(n, batch, prf)
    ctx = B.Context(table, early_termination=True)
    assert ctx.rows_per_leaf == 4
    ra, rb = ctx.eval(a, prf), ctx.eval(b, prf)
    assert reconstructs(ra, rb, table, alphas)
    check = min(batch, 4 if n >= 1 << 14 else 8)
    assert np.array_equal(ra[:check], et_oracle.eval_dot_et(orc, a[:check], prf, table))
    assert np.array_equal(ra, host_dot(a, prf, table))
    ctx.close()


@pytest.mark.parametrize("prf", PRFS)
def test_large_n(prf):
    n = 1 << 20
    table = random_table(n, 16, seed=3)
    a, b, alphas = keys_for(n, 64, prf)
    ctx = B.Context(table, early_termination=True)
    ra, rb = ctx.eval(a, prf), ctx.eval(b, prf)
    assert reconstructs(ra, rb, table, alphas)
    assert np.array_equal(ra[:16], host_dot(a[:16], prf, table))
    ctx.close()


def test_aes_n_2_24():
    n = 1 << 24
    table = random_table(n, 16, seed=4)
    a, b, alphas = keys_for(n, 32, B.PRF_AES128)
    ctx = B.Context(table, early_termination=True)
    ra, rb = ctx.eval(a, B.PRF_AES128), ctx.eval(b, B.PRF_AES128)
    assert reconstructs(ra, rb, table, alphas)
    assert np.array_equal(ra[:2], host_dot(a[:2], B.PRF_AES128, table))
    ctx.close()


KNOBS = [("subtree_log2", v) for v in range(1, 8)] + [
    ("one_launch", 0), ("frontier", 0), ("frontier_mb", 1), ("lane_split", 0), ("tma_rows", 1)]


@pytest.mark.parametrize("prf", (B.PRF_AES128, B.PRF_CHACHA20))
def test_knobs(prf):
    n = 1 << 14
    table = random_table(n, 16, seed=5)
    a, _, _ = keys_for(n, 40, prf)
    small = a[:3]
    ctx = B.Context(table, early_termination=True)
    want, want_small = ctx.eval(a, prf), ctx.eval(small, prf)
    assert np.array_equal(want, host_dot(a, prf, table))
    for name, value in KNOBS:
        c = B.Context(table, early_termination=True)
        c.set_option(name, value)
        assert np.array_equal(c.eval(a, prf), want), (name, value)
        assert np.array_equal(c.eval(small, prf), want_small), (name, value)
        c.close()
    ctx.close()


def test_leaf_cache_and_chunking():
    n, prf = 1 << 14, B.PRF_AES128
    table = random_table(n, 128, seed=6)
    a, _, _ = keys_for(n, 100, prf)
    want = host_dot(a, prf, table)
    for opts in ({}, {"leaf_cache": 0}, {"leaf_cache_mb": 2}, {"mac_tma": 0}):
        c = B.Context(table, early_termination=True)
        for k, v in opts.items():
            c.set_option(k, v)
        assert np.array_equal(c.eval(a, prf), want), opts
        c.close()


def test_key_paths():
    torch = pytest.importorskip("torch")
    n, prf, e = 1 << 12, B.PRF_SALSA20, 20
    table = random_table(n, e, seed=7)
    a, _, _ = keys_for(n, 45, prf)
    want = host_dot(a, prf, table)
    ctx = B.Context(table, early_termination=True)
    assert np.array_equal(ctx.eval(a, prf), want)
    pinned = C.POINTER(C.c_int32)()
    assert B.lib().b200dpf_host_staging(ctx.handle, len(a), C.byref(pinned)) == 0
    staged = np.ctypeslib.as_array(pinned, shape=(len(a) * 524,))
    staged[:] = a.reshape(-1)
    out = np.zeros((len(a), e), np.int32)
    assert B.lib().b200dpf_eval(ctx.handle, staged.reshape(len(a), 524).copy(), len(a), prf, out) == 0
    assert np.array_equal(out, want)
    assert np.array_equal(ctx.eval_gather(list(a), prf), want)
    packed = b"".join(B.key_pack_et(k) for k in a)
    assert np.array_equal(ctx.eval_packed(packed, len(a), prf), want)
    keys_dev = torch.from_numpy(a).cuda()
    out_dev = torch.zeros((len(a), e), dtype=torch.int32, device="cuda")
    ctx.eval_device(keys_dev.data_ptr(), len(a), prf, out_dev.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(out_dev.cpu().numpy(), want)
    base = torch.arange(len(a) * e, dtype=torch.int32, device="cuda").reshape(len(a), e)
    acc = base.clone()
    ctx.eval_device(keys_dev.data_ptr(), len(a), prf, acc.data_ptr(), accumulate=True)
    torch.cuda.synchronize()
    assert np.array_equal((acc - base).cpu().numpy(), want)
    ctx.close()


@pytest.mark.parametrize("g", (2, 4, 8))
def test_shards(g):
    n, prf, e = 1 << 12, B.PRF_AES128, 16
    table = random_table(n, e, seed=8)
    a, _, _ = keys_for(n, 9, prf)
    shares = np.stack([B.eval_cpu_et(k, prf) for k in a])
    whole = et_oracle.dot_u32(shares, table)
    total = np.zeros_like(whole, dtype=np.uint32)
    bits = g.bit_length() - 1
    for r in range(g):
        ctx = B.Context(table, shard_rank=r, shard_count=g, early_termination=True)
        part = ctx.eval(a, prf)
        val = int(format(r, "0%db" % bits)[::-1], 2)
        own = ((np.arange(n) >> 2) & (g - 1)) == val
        assert np.array_equal(part, et_oracle.dot_u32(shares[:, own], table[own])), r
        total += part.view(np.uint32)
        ctx.close()
    assert np.array_equal(total.view(np.int32), whole)


@pytest.mark.parametrize("prf", PRFS)
def test_expand(prf, orc):
    torch = pytest.importorskip("torch")
    n = 1 << 10
    table = random_table(n, 4, seed=9)
    a, _, _ = keys_for(n, 37, prf)
    ctx = B.Context(table, early_termination=True)
    keys_dev = torch.from_numpy(a).cuda()
    out = torch.zeros((len(a), n), dtype=torch.int32, device="cuda")
    ctx.expand_device(keys_dev.data_ptr(), len(a), prf, out.data_ptr())
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i in range(3):
        assert np.array_equal(got[i], et_oracle.eval_full_flat_et(orc, a[i], prf))
    assert np.array_equal(got, np.stack([B.eval_cpu_et(k, prf) for k in a]))
    ctx.close()


@pytest.mark.parametrize("g", (1, 4))
def test_row_updates(g):
    torch = pytest.importorskip("torch")
    n, prf, e = 1 << 12, B.PRF_CHACHA20, 24
    table = random_table(n, e, seed=10)
    a, _, _ = keys_for(n, 33, prf)
    rng = np.random.RandomState(11)
    idx = np.concatenate([rng.randint(0, n, 300), [5, 5, 6, 7, 4095, 4095]]).astype(np.int64)
    rows = rng.randint(-2**31, 2**31, size=(len(idx), e), dtype=np.int64).astype(np.int32)
    new = table.copy()
    for j, i in enumerate(idx):
        new[i] = rows[j]
    shares = np.stack([B.eval_cpu_et(k, prf) for k in a])
    bits = g.bit_length() - 1
    for path in ("host", "device"):
        total = np.zeros((len(a), e), np.uint32)
        for r in range(g):
            ctx = B.Context(table, shard_rank=r, shard_count=g, early_termination=True)
            if path == "host":
                ctx.update_rows(idx, rows)
            else:
                ti, tr = torch.from_numpy(idx).cuda(), torch.from_numpy(rows).cuda()
                ctx.update_rows_device(ti.data_ptr(), tr.data_ptr(), len(idx))
                torch.cuda.synchronize()
            part = ctx.eval(a, prf)
            val = int(format(r, "0%db" % bits)[::-1], 2) if bits else 0
            own = ((np.arange(n) >> 2) & (g - 1)) == val
            assert np.array_equal(part, et_oracle.dot_u32(shares[:, own], new[own])), (path, r)
            total += part.view(np.uint32)
            ctx.close()
        assert np.array_equal(total.view(np.int32), et_oracle.dot_u32(shares, new))


def test_kind_mismatch_and_introspection():
    n, prf = 1 << 10, B.PRF_AES128
    table = random_table(n, 16, seed=12)
    et_a, _, _ = keys_for(n, 3, prf)
    std_a, _ = B.gen_batch_secure(np.array([1, 2, 3], np.int64), n, bytes(44 * 3), prf)
    L = B.lib()
    et_ctx, std_ctx = B.Context(table, early_termination=True), B.Context(table)
    assert et_ctx.rows_per_leaf == 4 and std_ctx.rows_per_leaf == 1
    assert L.b200dpf_ctx_n(et_ctx.handle) == n
    out = np.zeros((3, 16), np.int32)
    assert L.b200dpf_eval(et_ctx.handle, np.ascontiguousarray(std_a), 3, prf, out) == EINVAL
    assert b"standard key" in L.b200dpf_last_error()
    assert L.b200dpf_eval(std_ctx.handle, np.ascontiguousarray(et_a), 3, prf, out) == EINVAL
    assert b"early-terminated" in L.b200dpf_last_error()
    ptrs = (C.c_void_p * 3)(*[k.ctypes.data for k in std_a])
    assert L.b200dpf_eval_gather(et_ctx.handle, ptrs, 3, prf, out) == EINVAL
    std_packed = b"".join(B.key_pack(k) for k in std_a)
    et_packed = b"".join(B.key_pack_et(k) for k in et_a)
    assert L.b200dpf_eval_packed(et_ctx.handle, std_packed, 3, prf, out) == EINVAL
    assert L.b200dpf_eval_packed(std_ctx.handle, et_packed, 3, prf, out) == EINVAL
    et_ctx.close()
    std_ctx.close()


def test_python_end_to_end():
    torch = pytest.importorskip("torch")
    import dpf
    for n, pad in ((1 << 12, False), (1000, True)):
        d = dpf.DPF(prf=dpf.DPF.PRF_AES128, early_termination=True, allow_non_pow2=pad)
        table = torch.randint(-2**31, 2**31 - 1, (n, 16), dtype=torch.int64).to(torch.int32)
        d.eval_init(table)
        idx = [0, 5, n - 1, 123, 77]
        pairs = [d.gen(k, n) for k in idx]
        ka, kb = [p[0] for p in pairs], [p[1] for p in pairs]
        ra, rb = d.eval_gpu(ka), d.eval_gpu(kb)
        assert torch.equal(ra - rb, table[idx])
        assert torch.equal(ra, d.eval_cpu(ka))
        assert torch.equal(d.eval_gpu(torch.stack(ka)), ra)
        assert torch.equal(d.eval_gpu_compact(d.pack_keys(ka)), ra)
        dev = d.eval_gpu_device(torch.stack(ka).cuda())
        assert torch.equal(dev.cpu(), ra)
        piped = list(d.eval_gpu_pipelined([torch.stack(ka), torch.stack(kb)]))
        assert torch.equal(piped[0], ra) and torch.equal(piped[1], rb)
        a, b = d.gen_batch(list(range(40)), d.table_num_entries)
        sh = d.expand_gpu_device(a.cuda())
        assert torch.equal(sh.cpu(), d.eval_cpu(a, one_hot_only=True))
        upd = torch.randint(-100, 100, (3, 16), dtype=torch.int32)
        d.update_rows([5, 123, 5], upd)
        assert torch.equal(d.eval_gpu(ka), d.eval_cpu(ka))
        assert torch.equal(d.eval_gpu(ka) - d.eval_gpu(kb), d.table[idx])
        d.close()
