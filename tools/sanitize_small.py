"""Small all-PRF run for compute-sanitizer (memcheck / racecheck / synccheck)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gpu-dpf_b200"))
import b200dpf  # noqa: E402

rng = np.random.RandomState(0)
for n, entry in ((512, 16), (2048, 40)):
    table = rng.randint(-2**31, 2**31, size=(n, entry), dtype=np.int64).astype(np.int32)
    ctx = b200dpf.Context(table)
    for prf in range(4):
        alphas = rng.randint(0, n, size=37)
        ka, kb = b200dpf.gen_batch(alphas, n, np.arange(37) + 5, prf)
        a, b = ctx.eval(ka, prf), ctx.eval(kb, prf)
        assert np.array_equal((a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32), table[alphas])
    packed = b"".join(b200dpf.key_pack(k) for k in ka)
    assert np.array_equal(ctx.eval_packed(packed, 37, 3), a)            # compact keys, last prf's batch
    assert np.array_equal(ctx.eval_gather(list(ka), 3), a)              # gather path
    if entry == 16:
        ctx.set_option("tma_rows", 1)                                      # TMA-staged rows variant (non-AES)
        ka2, kb2 = b200dpf.gen_batch(alphas, n, np.arange(37) + 5, 1)
        a2, b2 = ctx.eval(ka2, 1), ctx.eval(kb2, 1)
        assert np.array_equal((a2.astype(np.uint32) - b2.astype(np.uint32)).astype(np.int32), table[alphas])
    ctx.close()
# one-launch tree-top phase with more key groups (140) than AES blocks (132 on an H100 SXM): blocks take the
# host's per-block quota of 128-leaf items, then leave the balanced round by __syncthreads_and
n, nkeys = 256, 140 * 32
table = rng.randint(-2**31, 2**31, size=(n, 16), dtype=np.int64).astype(np.int32)
ctx = b200dpf.Context(table)
for name, value in (("subtree_log2", 1), ("top_log2", 7), ("balance_top", 1), ("one_launch", 1)):
    ctx.set_option(name, value)
alphas = rng.randint(0, n, size=nkeys)
ka, kb = b200dpf.gen_batch(alphas, n, np.arange(nkeys) + 9, 3)
a, b = ctx.eval(ka, 3), ctx.eval(kb, 3)
assert np.array_equal((a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32), table[alphas])
ctx.close()
# grouped (batch-PIR) launch
tables = [rng.randint(-2**31, 2**31, size=(m, 16), dtype=np.int64).astype(np.int32) for m in (256, 1024, 64)]
grp = b200dpf.GroupContext(tables)
bins = np.array([0, 1, 2, 1, 0, 1] * 8, np.int32)
alphas = np.array([rng.randint(0, tables[g].shape[0]) for g in bins])
ks = [b200dpf.gen(int(al), tables[g].shape[0], 77 + i, 2) for i, (al, g) in enumerate(zip(alphas, bins))]
ga = grp.eval(np.stack([k[0] for k in ks]), bins, 2)
gb = grp.eval(np.stack([k[1] for k in ks]), bins, 2)
assert np.array_equal((ga.astype(np.uint32) - gb.astype(np.uint32)).astype(np.int32), np.stack([tables[g][al] for g, al in zip(bins, alphas)]))
grp.close()
# grouped XOR-shared launch: blocks draw work units and reload a key group's words between units
tables = [rng.randint(-2**31, 2**31, size=(m, 20), dtype=np.int64).astype(np.int32) for m in (256, 4096, 1024)]
grp = b200dpf.GroupContext(tables, xor=True)
bins = np.array([0, 1, 2, 1, 1, 2, 1] * 7, np.int32)
alphas = np.array([rng.randint(0, tables[g].shape[0]) for g in bins], np.int64)
for prf in range(4):
    ka, kb = zip(*[b200dpf.gen_xor(int(al), tables[g].shape[0], bytes(range(i, i + 44)), prf)
                   for i, (al, g) in enumerate(zip(alphas, bins))])
    ga, gb = grp.eval(np.stack(ka), bins, prf), grp.eval(np.stack(kb), bins, prf)
    assert np.array_equal(ga ^ gb, np.stack([tables[g][al] for g, al in zip(bins, alphas)]))
grp.close()
# device-resident grouped evaluation, one context per kind: key gather, evaluation and result scatter on a
# caller's stream, two calls in flight (the second waits for the first's staging uploads only)
import torch  # noqa: E402
tables = [rng.randint(-2**31, 2**31, size=(m, 20), dtype=np.int64).astype(np.int32) for m in (256, 4096, 1024)]
bins = np.array([0, 1, 2, 1, 1, 2, 1] * 7, np.int32)
alphas = np.array([rng.randint(0, tables[g].shape[0]) for g in bins], np.int64)
for kw, gen in (({}, b200dpf.gen_batch_secure), ({"early_termination": True}, b200dpf.gen_batch_et),
                ({"xor": True}, b200dpf.gen_batch_xor)):
    grp = b200dpf.GroupContext(tables, **kw)
    ka, kb = np.zeros((len(bins), 524), np.int32), np.zeros((len(bins), 524), np.int32)
    for g in range(3):
        sel = np.nonzero(bins == g)[0]
        ka[sel], kb[sel] = gen(alphas[sel], tables[g].shape[0], bytes(range(44)) * len(sel), 2)
    stream = torch.cuda.Stream()
    keys = [torch.from_numpy(k).cuda() for k in (ka, kb)]
    outs = [torch.empty((len(bins), 20), dtype=torch.int32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    for k, o in zip(keys, outs):
        grp.eval_device(k.data_ptr(), bins, 2, o.data_ptr(), stream.cuda_stream)
    stream.synchronize()
    ga, gb = outs[0].cpu().numpy(), outs[1].cpu().numpy()
    assert np.array_equal(ga, grp.eval(ka, bins, 2)) and np.array_equal(gb, grp.eval(kb, bins, 2))
    rec = ga ^ gb if kw.get("xor") else (ga.astype(np.uint32) - gb.astype(np.uint32)).astype(np.int32)
    assert np.array_equal(rec, np.stack([tables[g][al] for g, al in zip(bins, alphas)]))
    grp.close()
# batch-PIR query batches, one context per kind, wire keys and compact queries: 5 queries of one key per bin,
# the second call of each format reusing the cached plan
nq = 5
qalphas = np.array([[rng.randint(0, t.shape[0]) for t in tables] for _ in range(nq)], np.int64)
for kw, gen in (({}, b200dpf.gen_batch_secure), ({"early_termination": True}, b200dpf.gen_batch_et),
                ({"xor": True}, b200dpf.gen_batch_xor)):
    grp = b200dpf.GroupContext(tables, **kw)
    ka, kb = np.zeros((nq, 3, 524), np.int32), np.zeros((nq, 3, 524), np.int32)
    for g in range(3):
        ka[:, g], kb[:, g] = gen(qalphas[:, g], tables[g].shape[0], bytes(range(44)) * nq, 2)
    tiled = np.tile(np.arange(3, dtype=np.int32), nq)
    for compact in (False, True):
        keys = [torch.from_numpy(grp.pack_queries(k) if compact else k).cuda() for k in (ka, kb)]
        outs = [torch.empty((nq, 3, 20), dtype=torch.int32, device="cuda") for _ in range(2)]
        torch.cuda.synchronize()
        for k, o in zip(keys, outs):
            grp.eval_queries_device(k.data_ptr(), nq, 2, o.data_ptr(), stream.cuda_stream, compact=compact)
        stream.synchronize()
        ga, gb = outs[0].cpu().numpy().reshape(-1, 20), outs[1].cpu().numpy().reshape(-1, 20)
        assert np.array_equal(ga, grp.eval(ka.reshape(-1, 524), tiled, 2))
        assert np.array_equal(gb, grp.eval(kb.reshape(-1, 524), tiled, 2))
        rec = ga ^ gb if kw.get("xor") else (ga.astype(np.uint32) - gb.astype(np.uint32)).astype(np.int32)
        assert np.array_equal(rec, np.stack([tables[g][al] for g, al in zip(tiled, qalphas.reshape(-1))]))
    grp.close()
# query batches generated on the GPU, one context per kind: the first call of the context generates (and uploads
# the per-bin table), compact queries of the same 5 x 3 pairs as above, evaluated on the same stream
qseeds = torch.from_numpy(np.frombuffer(bytes(range(44)) * nq * 3, np.uint8).copy()).cuda()
qalphas_dev = torch.from_numpy(qalphas).cuda()
for kw, gen in (({}, b200dpf.gen_batch_secure), ({"early_termination": True}, b200dpf.gen_batch_et),
                ({"xor": True}, b200dpf.gen_batch_xor)):
    grp = b200dpf.GroupContext(tables, **kw)
    qa, qb = [torch.empty(nq * grp.query_bytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
    outs = [torch.empty((nq, 3, 20), dtype=torch.int32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    grp.gen_queries_device(qalphas_dev.data_ptr(), qseeds.data_ptr(), nq, 2, qa.data_ptr(), qb.data_ptr(), stream.cuda_stream,
                           compact=True)
    for q, o in zip((qa, qb), outs):
        grp.eval_queries_device(q.data_ptr(), nq, 2, o.data_ptr(), stream.cuda_stream, compact=True)
    stream.synchronize()
    ka = np.zeros((nq, 3, 524), np.int32)
    for g in range(3):
        ka[:, g] = gen(qalphas[:, g], tables[g].shape[0], bytes(range(44)) * nq, 2)[0]
    assert np.array_equal(qa.cpu().numpy().reshape(nq, -1), grp.pack_queries(ka))
    ga, gb = outs[0].cpu().numpy(), outs[1].cpu().numpy()
    rec = ga ^ gb if kw.get("xor") else (ga.astype(np.uint32) - gb.astype(np.uint32)).astype(np.int32)
    assert np.array_equal(rec, np.stack([np.stack([tables[g][al] for g, al in enumerate(row)]) for row in qalphas]))
    grp.close()
# 4095 columns, one short of the widest entry: the leaf-cache pass and 64 MAC slices by both MAC kernels (the
# last slice 63 columns wide), an XOR-shared plain context (256 passes of 16 columns), and a grouped context
n, e = 1024, 4095
table = rng.randint(-2**31, 2**31, size=(n, e), dtype=np.int64).astype(np.int32)
alphas = rng.randint(0, n, size=40)
ka, kb = b200dpf.gen_batch(alphas, n, np.arange(40) + 3, 2)
ctx = b200dpf.Context(table)
for mac_tma in (1, 0):
    ctx.set_option("mac_tma", mac_tma)
    a, b = ctx.eval(ka, 2), ctx.eval(kb, 2)
    assert ctx.last_launches == 1 + 64
    assert np.array_equal((a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32), table[alphas])
ctx.close()
ka, kb = b200dpf.gen_batch_xor(alphas[:5], n, bytes(range(44)) * 5, 3)
ctx = b200dpf.Context(table, xor=True)
assert np.array_equal(ctx.eval(ka, 3) ^ ctx.eval(kb, 3), table[alphas[:5]])
ctx.close()
tables = [table[:256], table[:64]]
bins = np.array([0, 1, 1, 0, 1] * 4, np.int32)
alphas = np.array([rng.randint(0, tables[g].shape[0]) for g in bins], np.int64)
ka, kb = np.zeros((len(bins), 524), np.int32), np.zeros((len(bins), 524), np.int32)
for g in range(2):
    sel = np.nonzero(bins == g)[0]
    ka[sel], kb[sel] = b200dpf.gen_batch_et(alphas[sel], tables[g].shape[0], bytes(range(44)) * len(sel), 1)
grp = b200dpf.GroupContext(tables, early_termination=True)
ga, gb = grp.eval(ka, bins, 1), grp.eval(kb, bins, 1)
assert np.array_equal((ga.astype(np.uint32) - gb.astype(np.uint32)).astype(np.int32), table[alphas])
grp.close()
# one context, calls rotating over three streams with no host synchronisation between them: each larger batch
# grows the counters, tree-top tickets, frontier and (at 40 columns) the leaf cache while earlier calls may still
# run, so memcheck sees any use of scratch after it was freed; a row update on a fourth stream sits in the chain
n, e = 1024, 40
table = rng.randint(-2**31, 2**31, size=(n, e), dtype=np.int64).astype(np.int32)
alphas = rng.randint(0, n, size=600).astype(np.int64)
ka, kb = b200dpf.gen_batch_secure(alphas, n, bytes(range(44)) * 600, 2)
ctx = b200dpf.Context(table)
ctx.set_option("leaf_cache_mb", 1)
want = ctx.eval(ka, 2)
streams = [torch.cuda.Stream() for _ in range(4)]
keys = torch.from_numpy(ka).cuda()
batches = (1, 5, 33, 200, 600, 17)
outs = [torch.empty((b, e), dtype=torch.int32, device="cuda") for b in batches]
upd_idx = torch.from_numpy(np.array([alphas[0]], np.int64)).cuda()
upd_row = torch.from_numpy(table[alphas[0]][None].copy()).cuda()         # rewrites a row with its own value
torch.cuda.synchronize()
for i, (b, o) in enumerate(zip(batches, outs)):
    ctx.eval_device(keys.data_ptr(), b, 2, o.data_ptr(), stream=streams[i % 3].cuda_stream)
    if i == 3:
        ctx.update_rows_device(upd_idx.data_ptr(), upd_row.data_ptr(), 1, stream=streams[3].cuda_stream)
torch.cuda.synchronize()
for b, o in zip(batches, outs):
    assert np.array_equal(o.cpu().numpy(), want[:b])
rec = (want.astype(np.uint32) - ctx.eval(kb, 2).astype(np.uint32)).astype(np.int32)
assert np.array_equal(rec, table[alphas])
ctx.close()
# grouped evaluation from device-resident bins, planned on the GPU, one context per kind: histogram, sort, plan and
# list kernels, then the gather, evaluation and scatter; out-of-range bins mixed in, and a larger second batch that
# grows the plan's scratch while the first may still run
tables = [rng.randint(-2**31, 2**31, size=(m, 20), dtype=np.int64).astype(np.int32) for m in (256, 4096, 1024)]
bins = np.array([0, 1, 2, 1, 1, 2, 1] * 7, np.int32)
alphas = np.array([rng.randint(0, tables[g].shape[0]) for g in bins], np.int64)
for kw, gen in (({}, b200dpf.gen_batch_secure), ({"early_termination": True}, b200dpf.gen_batch_et),
                ({"xor": True}, b200dpf.gen_batch_xor)):
    grp = b200dpf.GroupContext(tables, **kw)
    ka, kb = np.zeros((len(bins), 524), np.int32), np.zeros((len(bins), 524), np.int32)
    for g in range(3):
        sel = np.nonzero(bins == g)[0]
        ka[sel], kb[sel] = gen(alphas[sel], tables[g].shape[0], bytes(range(44)) * len(sel), 3)
    with_bad = bins.copy()
    with_bad[[3, 10, 20]] = [-1, 3, 99]
    keys = [torch.from_numpy(k).cuda() for k in (ka, kb, ka)]
    bins_dev = [torch.from_numpy(b).cuda() for b in (bins[:20], bins, with_bad)]
    outs = [torch.empty((len(b), 20), dtype=torch.int32, device="cuda") for b in bins_dev]
    bad = torch.full((3,), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for i, (k, b, o) in enumerate(zip(keys, bins_dev, outs)):
        grp.eval_device_bins(k.data_ptr(), b.data_ptr(), len(b), 3, o.data_ptr(), bad[i:].data_ptr(), stream.cuda_stream)
    stream.synchronize()
    want_a, want_b = grp.eval(ka, bins, 3), grp.eval(kb, bins, 3)
    assert bad.cpu().tolist() == [0, 0, 3]
    assert np.array_equal(outs[0].cpu().numpy(), want_a[:20]) and np.array_equal(outs[1].cpu().numpy(), want_b)
    good = np.setdiff1d(np.arange(len(bins)), [3, 10, 20])
    assert np.array_equal(outs[2].cpu().numpy()[good], want_a[good]) and not outs[2].cpu().numpy()[[3, 10, 20]].any()
    rec = want_a ^ want_b if kw.get("xor") else (want_a.astype(np.uint32) - want_b.astype(np.uint32)).astype(np.int32)
    assert np.array_equal(rec, np.stack([tables[g][al] for g, al in zip(bins, alphas)]))
    grp.close()
print("sanitize run ok")
