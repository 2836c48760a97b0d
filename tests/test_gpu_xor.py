"""XOR-shared keys (128 table rows per GGM leaf, XOR results) on the GPU: every evaluation path of a
b200dpf_create_xor context, bit-exact against the per-index oracle (tests/xor_oracle.py) at small n and
against the host evaluation (itself checked against the oracle in test_xor_host.py) at large n."""
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
import oracle  # noqa: E402
import xor_oracle  # noqa: E402
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
    alphas[: min(batch, 6)] = [0, n - 1, 31, 32, 127, 128][: min(batch, 6)]
    seeds = rng.randint(0, 256, size=44 * batch).astype(np.uint8).tobytes()
    a, b = B.gen_batch_xor(alphas, n, seeds, prf)
    return a, b, alphas


def host_bits(keys, prf):
    return np.stack([xor_oracle.unpack_bits(B.eval_cpu_xor(k, prf)) for k in keys])


def host_result(keys, prf, table):
    return xor_oracle.xor_rows(host_bits(keys, prf), table)


def reconstructs(ra, rb, table, alphas):
    return np.array_equal((ra.view(np.uint32) ^ rb.view(np.uint32)).view(np.int32), table[alphas])


GRID = [  # (n, E, B): n from 2^8 to 2^20, entry sizes around the 16-column passes, batch sizes around the key quads
    (256, 1, 1), (256, 17, 3), (512, 5, 4), (1024, 16, 33), (1024, 200, 3), (1 << 12, 33, 5),
    (1 << 12, 32, 512), (1 << 14, 16, 512), (1 << 14, 128, 33), (1 << 14, 17, 1), (1 << 16, 16, 31), (1 << 16, 48, 17),
    (1 << 18, 16, 64), (1 << 20, 16, 2),
]


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("n,e,batch", GRID)
def test_bit_exact(prf, n, e, batch, orc):
    table = random_table(n, e, seed=n + e)
    a, b, alphas = keys_for(n, batch, prf)
    ctx = B.Context(table, xor=True)
    assert ctx.rows_per_leaf == 128
    ra, rb = ctx.eval(a, prf), ctx.eval(b, prf)
    assert reconstructs(ra, rb, table, alphas)
    if n <= 1 << 14:
        check = min(batch, 2 if n >= 1 << 12 else 4)
        assert np.array_equal(ra[:check], xor_oracle.eval_xor(orc, a[:check], prf, table))
    check = batch if n <= 1 << 16 else 4
    assert np.array_equal(ra[:check], host_result(a[:check], prf, table))
    ctx.close()


def test_aes_n_2_24():
    n = 1 << 24
    table = random_table(n, 16, seed=4)
    a, b, alphas = keys_for(n, 64, B.PRF_AES128)
    ctx = B.Context(table, xor=True)
    ra, rb = ctx.eval(a, B.PRF_AES128), ctx.eval(b, B.PRF_AES128)
    assert reconstructs(ra, rb, table, alphas)
    assert np.array_equal(ra[:2], host_result(a[:2], B.PRF_AES128, table))
    ctx.close()


def test_aes_n_2_26_sparse(orc):
    """n = 2^26, E = 20: 128-byte device rows, so the device table crosses the 4 GiB mark at device row 2^25.
    The device table is in breadth-first leaf order -- device row 128p + l holds natural row
    128 * bitrev_19(p) + l -- so the rows on both sides of that mark are derived from the permutation
    (device rows 2^25 .. are natural leaf 1, rows 128..; the rows just before it natural leaf 2^19 - 2).
    The table is zero except on a support set -- both sides of the 4 GiB mark and of the device table's
    end, both sides of natural leaf boundaries, the ends -- so the expected result is the XOR of the
    support rows whose share bit is set."""
    torch = pytest.importorskip("torch")
    n, e, prf = 1 << 26, 20, B.PRF_AES128
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs about 24 GiB of free device memory")
    depth = 26 - 7

    def natural(dev_row):
        leaf = int(format(dev_row >> 7, "0%db" % depth)[::-1], 2)
        return (leaf << 7) | (dev_row & 127)

    mark = (4 << 30) // 128                                    # device row at the 4 GiB byte offset
    at_mark = [natural(r) for r in (mark - 2, mark - 1, mark, mark + 1)]
    assert at_mark[2] == 128 and at_mark[1] == ((1 << depth) - 2) * 128 + 127
    support = set(at_mark) | {natural(r) for r in (n - 2, n - 1)}
    for c in (128, 256, 1 << 12, 1 << 20, 1 << 25, n // 2 + (1 << 24), n - 128):
        support.update((c - 2, c - 1, c, c + 1))
    support.update((0, 1, 127, n - 1))
    support = np.array(sorted(s for s in support if 0 <= s < n), np.int64)
    rng = np.random.RandomState(26)
    rows = rng.randint(-2**31, 2**31, size=(len(support), e), dtype=np.int64).astype(np.int32)
    table_dev = torch.zeros((n, e), dtype=torch.int32, device="cuda")
    table_dev[torch.from_numpy(support).cuda()] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    L = B.lib()
    h = C.c_void_p()
    assert L.b200dpf_create_xor(C.byref(h), C.c_void_p(table_dev.data_ptr()), n, e, 0, 0, 1) == 0, L.b200dpf_last_error()
    del table_dev
    alphas = np.array([at_mark[1], at_mark[2], 127, n - 1], np.int64)     # both sides of the 4 GiB mark
    seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
    a, b = B.gen_batch_xor(alphas, n, seeds, prf)
    out_a, out_b = np.zeros((4, e), np.int32), np.zeros((4, e), np.int32)
    assert L.b200dpf_eval(h, a, 4, prf, out_a) == 0
    assert L.b200dpf_eval(h, b, 4, prf, out_b) == 0
    L.b200dpf_destroy(h)
    rec = (out_a.view(np.uint32) ^ out_b.view(np.uint32)).view(np.int32)
    for k, alpha in enumerate(alphas):
        pos = np.searchsorted(support, alpha)
        assert rec[k].tolist() == rows[pos].tolist()          # every alpha is in the support set
    for k in range(2):
        bits = xor_oracle.unpack_bits(B.eval_cpu_xor(a[k], prf))[support]
        for j in range(0, len(support), 7):                   # spot checks against the per-index oracle
            assert int(bits[j]) == xor_oracle.share_bit(orc, a[k], int(support[j]), prf)
        assert np.array_equal(out_a[k], xor_oracle.xor_rows(bits, rows)[0])


KNOBS = [("subtree_log2", v) for v in range(1, 8)] + [
    ("one_launch", 0), ("frontier", 0), ("frontier_mb", 1), ("lane_split", 0), ("tma_rows", 1), ("leaf_cache", 0),
    ("mac_tma", 0), ("balance_top", 0), ("top_log2", 2), ("timing", 1), ("leaf_cache_mb", 1)]


@pytest.mark.parametrize("prf", (B.PRF_AES128, B.PRF_CHACHA20))
def test_knobs(prf):
    n = 1 << 14
    table = random_table(n, 20, seed=5)
    a, _, _ = keys_for(n, 40, prf)
    small = a[:3]
    ctx = B.Context(table, xor=True)
    want, want_small = ctx.eval(a, prf), ctx.eval(small, prf)
    assert np.array_equal(want, host_result(a, prf, table))
    assert np.array_equal(want_small, want[:3])
    for name, value in KNOBS:
        c = B.Context(table, xor=True)
        c.set_option(name, value)
        assert np.array_equal(c.eval(a, prf), want), (name, value)
        assert np.array_equal(c.eval(small, prf), want_small), (name, value)
        c.close()
    ctx.close()


def test_key_paths():
    torch = pytest.importorskip("torch")
    n, prf, e = 1 << 12, B.PRF_SALSA20, 20
    table = random_table(n, e, seed=7)
    a, _, _ = keys_for(n, 45, prf)
    want = host_result(a, prf, table)
    ctx = B.Context(table, xor=True)
    assert np.array_equal(ctx.eval(a, prf), want)
    pinned = C.POINTER(C.c_int32)()
    assert B.lib().b200dpf_host_staging(ctx.handle, len(a), C.byref(pinned)) == 0
    staged = np.ctypeslib.as_array(pinned, shape=(len(a) * 524,))
    staged[:] = a.reshape(-1)
    out = np.zeros((len(a), e), np.int32)
    assert B.lib().b200dpf_eval(ctx.handle, staged.reshape(len(a), 524).copy(), len(a), prf, out) == 0
    assert np.array_equal(out, want)
    assert np.array_equal(ctx.eval_gather(list(a), prf), want)
    packed = b"".join(B.key_pack_xor(k) for k in a)
    assert np.array_equal(ctx.eval_packed(packed, len(a), prf), want)
    keys_dev = torch.from_numpy(a).cuda()
    out_dev = torch.full((len(a), e), 7, dtype=torch.int32, device="cuda")
    ctx.eval_device(keys_dev.data_ptr(), len(a), prf, out_dev.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(out_dev.cpu().numpy(), want)
    # _eval_device_acc XORs into the destination
    base = torch.arange(len(a) * e, dtype=torch.int32, device="cuda").reshape(len(a), e) * 2654435761
    acc = base.clone()
    ctx.eval_device(keys_dev.data_ptr(), len(a), prf, acc.data_ptr(), accumulate=True)
    torch.cuda.synchronize()
    assert np.array_equal(torch.bitwise_xor(acc, base).cpu().numpy(), want)
    ctx.eval_device(keys_dev.data_ptr(), len(a), prf, acc.data_ptr(), accumulate=True)   # twice: back to base
    torch.cuda.synchronize()
    assert torch.equal(acc, base)
    ctx.close()


@pytest.mark.parametrize("g", (2, 4, 8))
def test_shards(g):
    n, prf, e = 1 << 12, B.PRF_AES128, 16
    table = random_table(n, e, seed=8)
    a, _, _ = keys_for(n, 9, prf)
    bits = host_bits(a, prf)
    whole = xor_oracle.xor_rows(bits, table)
    total = np.zeros_like(whole, dtype=np.uint32)
    nb = g.bit_length() - 1
    for r in range(g):
        ctx = B.Context(table, shard_rank=r, shard_count=g, xor=True)
        part = ctx.eval(a, prf)
        val = int(format(r, "0%db" % nb)[::-1], 2)
        own = ((np.arange(n) >> 7) & (g - 1)) == val
        assert np.array_equal(part, xor_oracle.xor_rows(bits[:, own], table[own])), r
        total ^= part.view(np.uint32)
        ctx.close()
    assert np.array_equal(total.view(np.int32), whole)


@pytest.mark.parametrize("prf", PRFS)
def test_expand(prf, orc):
    torch = pytest.importorskip("torch")
    n = 1 << 12
    table = random_table(n, 4, seed=9)
    a, _, _ = keys_for(n, 37, prf)
    ctx = B.Context(table, xor=True)
    keys_dev = torch.from_numpy(a).cuda()
    out = torch.zeros((len(a), n // 32), dtype=torch.int32, device="cuda")
    ctx.expand_device(keys_dev.data_ptr(), len(a), prf, out.data_ptr())
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(np.uint32)
    for i in range(2):
        assert np.array_equal(got[i], xor_oracle.pack_bits(xor_oracle.share_bits(orc, a[i], prf)))
    assert np.array_equal(got, np.stack([B.eval_cpu_xor(k, prf) for k in a]))
    ctx.close()


@pytest.mark.parametrize("g", (1, 4))
def test_row_updates(g):
    torch = pytest.importorskip("torch")
    n, prf, e = 1 << 12, B.PRF_CHACHA20, 24
    table = random_table(n, e, seed=10)
    a, _, _ = keys_for(n, 33, prf)
    rng = np.random.RandomState(11)
    # duplicates, the last row of a leaf and the first of the next, both ends
    idx = np.concatenate([rng.randint(0, n, 300), [5, 5, 127, 128, 127, 255, 256, 4095, 4095, 0]]).astype(np.int64)
    rows = rng.randint(-2**31, 2**31, size=(len(idx), e), dtype=np.int64).astype(np.int32)
    new = table.copy()
    for j, i in enumerate(idx):
        new[i] = rows[j]
    bits = host_bits(a, prf)
    nb = g.bit_length() - 1
    for path in ("host", "device"):
        total = np.zeros((len(a), e), np.uint32)
        for r in range(g):
            ctx = B.Context(table, shard_rank=r, shard_count=g, xor=True)
            if path == "host":
                ctx.update_rows(idx, rows)
            else:
                ti, tr = torch.from_numpy(idx).cuda(), torch.from_numpy(rows).cuda()
                ctx.update_rows_device(ti.data_ptr(), tr.data_ptr(), len(idx))
                torch.cuda.synchronize()
            part = ctx.eval(a, prf)
            val = int(format(r, "0%db" % nb)[::-1], 2) if nb else 0
            own = ((np.arange(n) >> 7) & (g - 1)) == val
            assert np.array_equal(part, xor_oracle.xor_rows(bits[:, own], new[own])), (path, r)
            total ^= part.view(np.uint32)
            ctx.close()
        assert np.array_equal(total.view(np.int32), xor_oracle.xor_rows(bits, new))


def test_kind_mismatch_and_introspection():
    n, prf = 1 << 10, B.PRF_AES128
    table = random_table(n, 16, seed=12)
    xk, _, _ = keys_for(n, 3, prf)
    al = np.array([1, 2, 3], np.int64)
    std_a, _ = B.gen_batch_secure(al, n, bytes(44 * 3), prf)
    et_a, _ = B.gen_batch_et(al, n, bytes(44 * 3), prf)
    L = B.lib()
    x_ctx, et_ctx, std_ctx = B.Context(table, xor=True), B.Context(table, early_termination=True), B.Context(table)
    assert x_ctx.rows_per_leaf == 128 and et_ctx.rows_per_leaf == 4 and std_ctx.rows_per_leaf == 1
    assert L.b200dpf_ctx_n(x_ctx.handle) == n and L.b200dpf_ctx_entry_size(x_ctx.handle) == 16
    out = np.zeros((3, 16), np.int32)
    for keys, word in ((std_a, b"standard key"), (et_a, b"early-terminated key")):
        assert L.b200dpf_eval(x_ctx.handle, np.ascontiguousarray(keys), 3, prf, out) == EINVAL
        assert word in L.b200dpf_last_error()
        ptrs = (C.c_void_p * 3)(*[k.ctypes.data for k in keys])
        assert L.b200dpf_eval_gather(x_ctx.handle, ptrs, 3, prf, out) == EINVAL
    for ctx in (et_ctx, std_ctx):
        assert L.b200dpf_eval(ctx.handle, np.ascontiguousarray(xk), 3, prf, out) == EINVAL
        assert b"XOR-shared key" in L.b200dpf_last_error()
    x_packed = b"".join(B.key_pack_xor(k) for k in xk)
    assert L.b200dpf_eval_packed(x_ctx.handle, b"".join(B.key_pack(k) for k in std_a), 3, prf, out) == EINVAL
    assert L.b200dpf_eval_packed(x_ctx.handle, b"".join(B.key_pack_et(k) for k in et_a), 3, prf, out) == EINVAL
    assert L.b200dpf_eval_packed(et_ctx.handle, x_packed, 3, prf, out) == EINVAL
    assert L.b200dpf_eval_packed(std_ctx.handle, x_packed, 3, prf, out) == EINVAL
    assert np.array_equal(x_ctx.eval_packed(x_packed, 3, prf), x_ctx.eval(xk, prf))
    for c in (x_ctx, et_ctx, std_ctx):
        c.close()


def test_python_end_to_end():
    torch = pytest.importorskip("torch")
    import dpf
    for n, pad in ((1 << 12, False), (1000, True)):
        d = dpf.DPF(prf=dpf.DPF.PRF_AES128, xor=True, allow_non_pow2=pad)
        table = torch.randint(-2**31, 2**31 - 1, (n, 16), dtype=torch.int64).to(torch.int32)
        d.eval_init(table)
        idx = [0, 5, n - 1, 123, 127, 128]
        pairs = [d.gen(k, n) for k in idx]
        ka, kb = [p[0] for p in pairs], [p[1] for p in pairs]
        ra, rb = d.eval_gpu(ka), d.eval_gpu(kb)
        assert torch.equal(torch.bitwise_xor(ra, rb), table[idx])
        assert torch.equal(ra, d.eval_cpu(ka))
        assert torch.equal(d.eval_gpu(torch.stack(ka)), ra)
        assert torch.equal(d.eval_gpu_compact(d.pack_keys(ka)), ra)
        dev = d.eval_gpu_device(torch.stack(ka).cuda())
        assert torch.equal(dev.cpu(), ra)
        a, b = d.gen_batch(list(range(40)), d.table_num_entries)
        sh = d.expand_gpu_device(a.cuda())
        bits = ((sh.cpu().view(-1, 1) >> torch.arange(32, dtype=torch.int32)) & 1).reshape(40, -1)
        assert torch.equal(bits, d.eval_cpu(a, one_hot_only=True))
        upd = torch.randint(-100, 100, (3, 16), dtype=torch.int32)
        d.update_rows([5, 123, 5], upd)
        assert torch.equal(d.eval_gpu(ka), d.eval_cpu(ka))
        assert torch.equal(torch.bitwise_xor(d.eval_gpu(ka), d.eval_gpu(kb)), d.table[idx])
        d.close()
    # the multi-device pieces are refused up front
    with pytest.raises(Exception):
        dpf.DPF(devices=[0, 1], xor=True)


def test_dpf_cpp_surface():
    torch = pytest.importorskip("torch")
    import dpf_cpp
    n, prf = 1 << 10, B.PRF_CHACHA20
    table = torch.randint(-2**31, 2**31 - 1, (n, 16), dtype=torch.int64).to(torch.int32)
    buf = dpf_cpp.eval_init_xor(table)
    a, b = dpf_cpp.gen_xor(300, n, bytes(range(44)), prf)
    ra = dpf_cpp.eval_gpu_packed(torch.stack([a]), buf, prf)
    rb = dpf_cpp.eval_gpu_packed(torch.stack([b]), buf, prf)
    assert torch.equal(torch.bitwise_xor(ra, rb)[0], table[300])
    assert torch.equal(dpf_cpp.key_unpack_xor(dpf_cpp.key_pack_xor(a)), a)
    assert dpf_cpp.rows_per_leaf(buf) == 128
    dpf_cpp.eval_free(buf)
