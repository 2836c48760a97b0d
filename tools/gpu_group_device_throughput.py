"""End-to-end cost of a grouped (batch-PIR) evaluation: the host path against the device-resident path.

    python tools/gpu_group_device_throughput.py [--reps 3] [--calls 20] [--out gpu_group_device_throughput.json]

Shapes are (bins, log2 rows per bin, queries, columns), one key per (query, bin), all pairs in one call: those
of DESIGN.md section 10.1.  XOR-shared and early-terminated keys run every shape, standard keys two, each with
AES and ChaCha20.  Per shape, kind and PRF three ways run in turn, `reps` rounds each, in one process:
    host      b200dpf_group_eval: host keys in, host results out; wall clock per call, each call ends in
              its own synchronisation (key checks, packing, upload, launch, download, reorder)
    device    b200dpf_group_eval_device: `calls` calls enqueued back to back on one stream, keys already on the
              device; CUDA events around all of them, divided by `calls`
    pipelined a server loop: host keys (pinned, wire format) uploaded by the caller on a copy stream, evaluated
              with b200dpf_group_eval_device on a compute stream, results downloaded on a third stream into
              pinned memory, two batches in flight (what DPF.eval_gpu_pipelined does for plain contexts);
              wall clock of `calls` batches after one warm-up batch, divided by `calls`
and b200dpf_ctx_last_device_ms (the evaluation launches alone) after the host and the device calls.  Reported
times are medians of the rounds.  Every timed batch is checked: the calls alternate the two servers' keys, and
every (a, b) pair of results reconstructs table[bin][alpha] (a - b, or a ^ b).  The gather and scatter
kernels' own times come from torch.profiler over a few device calls, beside the bytes each one moves.  The
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
KINDS = {"xor": (B.gen_batch_xor, {"xor": True}, 7), "et": (B.gen_batch_et, {"early_termination": True}, 2),
         "std": (B.gen_batch_secure, {}, 0)}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def make_pairs(kind, nbins, n, queries, prf, seed):
    """one key pair per (query, bin), query-major: pair q * nbins + g is for bin g"""
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=queries * nbins).astype(np.int64)
    seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
    a, b = KINDS[kind][0](alphas, n, seeds, prf)
    return a, b, np.tile(np.arange(nbins, dtype=np.int32), queries), alphas


def reconstructs(kind, ra, rb, want):
    if kind == "xor":
        return np.array_equal((ra.view(np.uint32) ^ rb.view(np.uint32)).view(np.int32), want)
    return np.array_equal((ra.view(np.uint32) - rb.view(np.uint32)).view(np.int32), want)


def run_host(ctx, keys, bins, prf, calls, kind, want):
    times, ok, outs = [], True, []
    for i in range(calls):
        t0 = time.perf_counter()
        outs.append(ctx.eval(keys[i % 2], bins, prf))
        times.append((time.perf_counter() - t0) * 1e3)
        if i % 2 == 1:
            ok = ok and reconstructs(kind, outs[0], outs[1], want)
            outs = []
    return statistics.median(times), ctx.last_device_ms, ok


def run_device(ctx, keys_dev, bins, prf, outs, kind, want):
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i, o in enumerate(outs):
        ctx.eval_device(keys_dev[i % 2].data_ptr(), bins, prf, o.data_ptr(), stream.cuda_stream)
    e1.record(stream)
    e1.synchronize()
    per_call = e0.elapsed_time(e1) / len(outs)
    dev_ms = ctx.last_device_ms
    ok = True
    for i in range(0, len(outs) - 1, 2):
        ok = ok and reconstructs(kind, outs[i].cpu().numpy(), outs[i + 1].cpu().numpy(), want)
    return per_call, dev_ms, ok


def run_pipelined(ctx, keys_host, bins, prf, calls, kind, want, e):
    """keys_host: two pinned int32 [B, 524] tensors; two batches in flight"""
    dev = torch.device("cuda", 0)
    compute, h2d, d2h = torch.cuda.Stream(dev), torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    depth = 2
    kbuf = [torch.empty(keys_host[0].shape, dtype=torch.int32, device=dev) for _ in range(depth)]
    obuf = [torch.empty((keys_host[0].shape[0], e), dtype=torch.int32, device=dev) for _ in range(depth)]
    hout = [torch.empty((keys_host[0].shape[0], e), dtype=torch.int32, pin_memory=True) for _ in range(calls + 1)]
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
        ctx.eval_device(kbuf[s].data_ptr(), bins, prf, obuf[s].data_ptr(), compute.cuda_stream)
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


def io_kernel_times(ctx, keys_dev, bins, prf, out):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ctx.eval_device(keys_dev.data_ptr(), bins, prf, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    t = {}
    for ev in prof.key_averages():
        for k in ("gather", "scatter"):
            if "group_%s_kernel" % k in ev.key and ev.count:
                total = getattr(ev, "device_time_total", None)
                t[k] = (total if total is not None else ev.cuda_time_total) / ev.count / 1e3     # us -> ms
    return {k: t.get(k) for k in ("gather", "scatter")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default="gpu_group_device_throughput.json")
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
        for prf in (B.PRF_AES128, B.PRF_CHACHA20):
            a, b, bins, alphas = make_pairs(kind, nbins, n, queries, prf, seed=nbins * 7 + lg + prf)
            want = np.stack([tables[g][x] for g, x in zip(bins, alphas)])
            keys_dev = [torch.from_numpy(k).cuda() for k in (a, b)]
            keys_pin = [torch.from_numpy(k).pin_memory() for k in (a, b)]
            outs = [torch.empty((len(bins), e), dtype=torch.int32, device="cuda") for _ in range(args.calls)]
            ctx.eval(a, bins, prf)                                        # warm-up of both paths
            run_device(ctx, keys_dev, bins, prf, outs[:2], kind, want)
            res = {"host": [], "host_dev": [], "device": [], "device_dev": [], "pipelined": []}
            ok = True
            for _ in range(args.reps):
                h, hd, o1 = run_host(ctx, (a, b), bins, prf, 6, kind, want)
                d, dd, o2 = run_device(ctx, keys_dev, bins, prf, outs, kind, want)
                p, o3 = run_pipelined(ctx, keys_pin, bins, prf, args.calls, kind, want, e)
                ok = ok and o1 and o2 and o3
                for k, v in zip(res, (h, hd, d, dd, p)):
                    res[k].append(v)
            io = io_kernel_times(ctx, keys_dev[0], bins, prf, outs[0])
            depth = lg - KINDS[kind][2]
            pairs = len(bins)
            row = {"kind": kind, "prf": NAMES[prf], "bins": nbins, "rows": n, "queries": queries, "E": e, "pairs": pairs,
                   "ok": bool(ok), **{k + "_ms": statistics.median(v) for k, v in res.items()},
                   "gather_ms": io["gather"], "scatter_ms": io["scatter"],
                   "gather_bytes": 2 * pairs * (32 + 64 * depth) + 8 * pairs, "scatter_bytes": 2 * pairs * 4 * e + 8 * pairs,
                   "h2d_bytes_pipelined": pairs * 2096}
            row["device_speedup"] = row["host_ms"] / row["device_ms"]
            row["pipelined_speedup"] = row["host_ms"] / row["pipelined_ms"]
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
