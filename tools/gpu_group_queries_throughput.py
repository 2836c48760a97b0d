"""Batch-PIR query batches: b200dpf_group_eval_queries_device (wire keys and compact queries) against
b200dpf_group_eval_device with the bins tiled.

    python tools/gpu_group_queries_throughput.py [--reps 3] [--calls 20] [--out gpu_group_queries_throughput.json]

Shapes are (bins, log2 rows per bin, queries, columns), one key per (query, bin): those of DESIGN.md section 8's
device-path table.  XOR-shared and early-terminated keys run every shape, standard keys two, each with AES and
ChaCha20.  Per shape, kind and PRF the ways below run in turn, `reps` rounds each, in one process:
    device    b200dpf_group_eval_device, wire keys and the bins 0 .. nbins-1 tiled per query (sort, plan and
              order list on the host every call)
    wire      b200dpf_group_eval_queries_device, the same wire keys (plan cached after the first call)
    compact   b200dpf_group_eval_queries_device on compact queries (GroupContext.pack_queries)
Each way makes `calls` calls back to back on one stream with the keys already on the device.  "host" is the
median wall clock around one call (the time the caller's thread spends in it, enqueue only), "per call" is CUDA
events around all the calls divided by `calls`, and "launches" is b200dpf_ctx_last_device_ms (the evaluation
launches alone).  Then a server loop, "pipelined": host keys in pinned memory uploaded on a copy stream,
evaluated on a compute stream, results downloaded on a third stream into pinned memory, two batches in flight,
wall clock of `calls` batches after one warm-up batch divided by `calls`; once with wire keys into
b200dpf_group_eval_device and once with compact queries into b200dpf_group_eval_queries_device, with the bytes
each uploads per batch.  Reported times are medians of the rounds.  Every timed batch is checked: the calls
alternate the two servers' keys, and every (a, b) pair reconstructs table[bin][alpha] (a - b, or a ^ b).  The
card, its power limit and SM clock are read in the same run (nvidia-smi, read-only queries).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gpu-dpf_b200")]
import b200dpf as B  # noqa: E402

NAMES = {B.PRF_AES128: "AES128", B.PRF_CHACHA20: "CHACHA20"}
SHAPES = [(64, 12, 256, 16), (256, 10, 256, 16), (16, 14, 512, 16), (64, 12, 32, 16), (1024, 10, 64, 16),
          (64, 12, 256, 40)]
STD_SHAPES = [(64, 12, 256, 16), (1024, 10, 64, 16)]
KINDS = {"xor": (B.gen_batch_xor, {"xor": True}), "et": (B.gen_batch_et, {"early_termination": True}),
         "std": (B.gen_batch_secure, {})}
WAYS = ("device", "wire", "compact")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def make_queries(kind, nbins, n, queries, prf, seed):
    """one key pair per (query, bin): int32 [queries, nbins, 524] twice, and the alphas [queries, nbins]"""
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=queries * nbins).astype(np.int64)
    seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
    a, b = KINDS[kind][0](alphas, n, seeds, prf)
    shape = (queries, nbins, B.KEY_WORDS)
    return a.reshape(shape), b.reshape(shape), alphas.reshape(queries, nbins)


def reconstructs(kind, ra, rb, want):
    ra, rb = ra.reshape(want.shape), rb.reshape(want.shape)
    if kind == "xor":
        return np.array_equal((ra.view(np.uint32) ^ rb.view(np.uint32)).view(np.int32), want)
    return np.array_equal((ra.view(np.uint32) - rb.view(np.uint32)).view(np.int32), want)


def call(ctx, way, keys_ptr, bins, queries, prf, out_ptr, stream):
    if way == "device":
        ctx.eval_device(keys_ptr, bins, prf, out_ptr, stream)
    else:
        ctx.eval_queries_device(keys_ptr, queries, prf, out_ptr, stream, compact=way == "compact")


def run_calls(ctx, way, keys_dev, bins, queries, prf, outs, kind, want):
    """`len(outs)` calls back to back on one stream: median host time per call, device time per call,
    last_device_ms, all pairs reconstructed"""
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    host = []
    e0.record(stream)
    for i, o in enumerate(outs):
        t0 = time.perf_counter()
        call(ctx, way, keys_dev[i % 2].data_ptr(), bins, queries, prf, o.data_ptr(), stream.cuda_stream)
        host.append((time.perf_counter() - t0) * 1e3)
    e1.record(stream)
    e1.synchronize()
    ok = all(reconstructs(kind, outs[i].cpu().numpy(), outs[i + 1].cpu().numpy(), want) for i in range(0, len(outs) - 1, 2))
    return statistics.median(host), e0.elapsed_time(e1) / len(outs), ctx.last_device_ms, ok


def run_pipelined(ctx, way, keys_host, bins, queries, prf, calls, kind, want, e):
    """keys_host: two pinned tensors (wire keys for "device", compact queries for "compact"); two batches in flight"""
    dev = torch.device("cuda", 0)
    compute, h2d, d2h = torch.cuda.Stream(dev), torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    depth = 2
    nout = want.size
    kbuf = [torch.empty(keys_host[0].shape, dtype=keys_host[0].dtype, device=dev) for _ in range(depth)]
    obuf = [torch.empty(nout, dtype=torch.int32, device=dev) for _ in range(depth)]
    hout = [torch.empty(nout, dtype=torch.int32, pin_memory=True) for _ in range(calls + 1)]
    free = [torch.cuda.Event() for _ in range(depth)]     # slot reusable: its download is done
    done = []
    torch.cuda.synchronize()
    t0 = None
    for i in range(calls + 1):                            # batch 0 warms up
        if i == 1:
            done[0].synchronize()
            t0 = time.perf_counter()
        s = i % depth
        h2d.wait_event(free[s])
        with torch.cuda.stream(h2d):
            kbuf[s].copy_(keys_host[i % 2], non_blocking=True)
            up = torch.cuda.Event()
            up.record(h2d)
        compute.wait_event(up)
        call(ctx, way, kbuf[s].data_ptr(), bins, queries, prf, obuf[s].data_ptr(), compute.cuda_stream)
        ev = torch.cuda.Event()
        ev.record(compute)
        d2h.wait_event(ev)
        with torch.cuda.stream(d2h):
            hout[i].copy_(obuf[s], non_blocking=True)
            fin = torch.cuda.Event()
            fin.record(d2h)
        free[s] = fin
        done.append(fin)
    done[-1].synchronize()
    per_batch = (time.perf_counter() - t0) * 1e3 / calls
    ok = reconstructs(kind, hout[0].numpy(), hout[1].numpy(), want)
    ok = ok and all(torch.equal(hout[i], hout[i % 2]) for i in range(2, calls + 1))
    return per_batch, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default="gpu_group_queries_throughput.json")
    args = ap.parse_args()
    info = card()
    print("card:", info, flush=True)
    rows = []
    cases = [(k, sh) for sh in SHAPES for k in ("xor", "et")] + [("std", sh) for sh in STD_SHAPES]
    for kind, (nbins, lg, queries, e) in cases:
        n = 1 << lg
        tables = [np.random.RandomState(1000 + g).randint(-2**31, 2**31, size=(n, e), dtype=np.int64).astype(np.int32)
                  for g in range(nbins)]
        ctx = B.GroupContext(tables, **KINDS[kind][1])
        bins = np.tile(np.arange(nbins, dtype=np.int32), queries)
        for prf in (B.PRF_AES128, B.PRF_CHACHA20):
            a, b, alphas = make_queries(kind, nbins, n, queries, prf, seed=nbins * 7 + lg + prf)
            want = np.stack([np.stack([tables[g][x] for g, x in enumerate(row)]) for row in alphas])
            packed = [ctx.pack_queries(k) for k in (a, b)]
            keys = {"device": (a, b), "wire": (a, b), "compact": packed}
            keys_dev = {w: [torch.from_numpy(k).cuda() for k in keys[w]] for w in WAYS}
            keys_pin = {w: [torch.from_numpy(k).pin_memory() for k in keys[w]] for w in ("device", "compact")}
            outs = [torch.empty((queries, nbins, e), dtype=torch.int32, device="cuda") for _ in range(args.calls)]
            for w in WAYS:                                                # warm-up: every way plans its shape
                run_calls(ctx, w, keys_dev[w], bins, queries, prf, outs[:2], kind, want)
            res = {k: [] for k in ("%s_%s" % (w, m) for w in WAYS for m in ("host_ms", "per_call_ms", "launches_ms"))}
            res.update(pipelined_wire_ms=[], pipelined_compact_ms=[])
            ok = True
            for _ in range(args.reps):
                for w in WAYS:
                    h, d, dd, o = run_calls(ctx, w, keys_dev[w], bins, queries, prf, outs, kind, want)
                    ok = ok and o
                    for m, v in zip(("host_ms", "per_call_ms", "launches_ms"), (h, d, dd)):
                        res["%s_%s" % (w, m)].append(v)
                for w, name in (("device", "pipelined_wire_ms"), ("compact", "pipelined_compact_ms")):
                    p, o = run_pipelined(ctx, w, keys_pin[w], bins, queries, prf, args.calls, kind, want, e)
                    ok = ok and o
                    res[name].append(p)
            pairs = queries * nbins
            row = {"kind": kind, "prf": NAMES[prf], "bins": nbins, "rows": n, "queries": queries, "E": e, "pairs": pairs,
                   "ok": bool(ok), **{k: statistics.median(v) for k, v in res.items()},
                   "h2d_bytes_wire": pairs * B.KEY_WORDS * 4, "h2d_bytes_compact": queries * ctx.query_bytes}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del keys_dev, keys_pin, outs
        ctx.close()
    out = {"card": info, "reps": args.reps, "calls": args.calls, "rows": rows}
    path = args.out if os.path.isabs(args.out) else os.path.join(os.getcwd(), args.out)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("all ok" if all(r["ok"] for r in rows) else "CHECK FAILED")


if __name__ == "__main__":
    main()
