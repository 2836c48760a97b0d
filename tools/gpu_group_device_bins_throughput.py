"""Grouped evaluation with the bins on the device, planned on the GPU (b200dpf_group_eval_device_bins), against
b200dpf_group_eval_device, which takes the bins on the host and plans there, on the same keys and bins.

    python tools/gpu_group_device_bins_throughput.py [--reps 3] [--calls 20] [--out gpu_group_device_bins_throughput.json]

Shapes are (bins, log2 rows per bin, keys per bin on average, columns): those of DESIGN.md section 8's device-path
table.  XOR-shared and early-terminated keys run every shape, standard keys two, each with AES and ChaCha20, and each
with two bin lists of the same length: "random" (every key's bin drawn uniformly) and "tiled" (0 .. nbins-1 repeated,
the batch-PIR shape).  Per case the two ways run in turn, `reps` rounds each, in one process:
    host_bins    b200dpf_group_eval_device, bins on the host (sort, plan and order list on the caller's thread)
    device_bins  b200dpf_group_eval_device_bins, bins on the device (histogram, sort, plan and lists on the GPU)
Each way makes `calls` calls back to back on one stream with keys and bins already on the device.  "host" is the
median wall clock around one call (the time the caller's thread spends in it), "per call" is CUDA events around all
the calls divided by `calls`, and "launches" is b200dpf_ctx_last_device_ms (the evaluation launches alone).  Reported
times are medians of the rounds.  "plan kernels" is the device time of device_bins' plan (the histogram's memset, the
histogram, the radix sort, the order, plan and list kernels) per call, summed from a torch.profiler trace of
`calls` further calls taken after the timed rounds.  Every timed batch is checked: the calls alternate the two
servers' keys, and every (a, b) pair reconstructs table[bin][alpha] (a - b, or a ^ b).  The card, its power limit and
SM clock are read in the same run (nvidia-smi, read-only queries).
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
WAYS = ("host_bins", "device_bins")
PLAN_KERNELS = ("group_hist_kernel", "group_order_kernel", "group_plan_kernel", "group_emit_kernel", "DeviceRadixSort")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def reconstructs(kind, ra, rb, want):
    if kind == "xor":
        return np.array_equal((ra.view(np.uint32) ^ rb.view(np.uint32)).view(np.int32), want)
    return np.array_equal((ra.view(np.uint32) - rb.view(np.uint32)).view(np.int32), want)


def call(ctx, way, keys_ptr, bins, bins_dev, prf, out_ptr, stream):
    if way == "host_bins":
        ctx.eval_device(keys_ptr, bins, prf, out_ptr, stream)
    else:
        ctx.eval_device_bins(keys_ptr, bins_dev.data_ptr(), len(bins), prf, out_ptr, 0, stream)


def run_calls(ctx, way, keys_dev, bins, bins_dev, prf, outs, kind, want):
    """`len(outs)` calls back to back on one stream: median host time per call, device time per call,
    last_device_ms, all pairs reconstructed"""
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    host = []
    e0.record(stream)
    for i, o in enumerate(outs):
        t0 = time.perf_counter()
        call(ctx, way, keys_dev[i % 2].data_ptr(), bins, bins_dev, prf, o.data_ptr(), stream.cuda_stream)
        host.append((time.perf_counter() - t0) * 1e3)
    e1.record(stream)
    e1.synchronize()
    ok = all(reconstructs(kind, outs[i].cpu().numpy(), outs[i + 1].cpu().numpy(), want) for i in range(0, len(outs) - 1, 2))
    return statistics.median(host), e0.elapsed_time(e1) / len(outs), ctx.last_device_ms, ok


def plan_kernel_ms(ctx, keys_dev, bins, bins_dev, prf, outs):
    """device time per call of device_bins' plan kernels, from a profiler trace of len(outs) calls"""
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i, o in enumerate(outs):
            call(ctx, "device_bins", keys_dev[i % 2].data_ptr(), bins, bins_dev, prf, o.data_ptr(), stream.cuda_stream)
        stream.synchronize()
    total_us, memset_us = 0.0, 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if any(k in ev.key for k in PLAN_KERNELS):
            total_us += t
        elif "Memset" in ev.key or "memset" in ev.key:
            memset_us += t
    # the histogram's clear is the only memset of a warm call: the evaluation clears its results and tickets in-kernel
    return (total_us + memset_us) / 1e3 / len(outs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default="gpu_group_device_bins_throughput.json")
    args = ap.parse_args()
    info = card()
    print("card:", info, flush=True)
    rows = []
    cases = [(k, sh) for sh in SHAPES for k in ("xor", "et")] + [("std", sh) for sh in STD_SHAPES]
    for kind, (nbins, lg, per_bin, e) in cases:
        n = 1 << lg
        tables = [np.random.RandomState(1000 + g).randint(-2**31, 2**31, size=(n, e), dtype=np.int64).astype(np.int32)
                  for g in range(nbins)]
        ctx = B.GroupContext(tables, **KINDS[kind][1])
        pairs = nbins * per_bin
        for prf in (B.PRF_AES128, B.PRF_CHACHA20):
            rng = np.random.RandomState(nbins * 7 + lg + prf)
            alphas = rng.randint(0, n, size=pairs).astype(np.int64)
            seeds = rng.randint(0, 256, size=44 * pairs).astype(np.uint8).tobytes()
            a, b = KINDS[kind][0](alphas, n, seeds, prf)        # every bin has n rows: a key fits any bin
            keys_dev = [torch.from_numpy(k).cuda() for k in (a, b)]
            outs = [torch.empty((pairs, e), dtype=torch.int32, device="cuda") for _ in range(args.calls)]
            for mix in ("random", "tiled"):
                bins = (rng.randint(0, nbins, size=pairs) if mix == "random" else np.tile(np.arange(nbins), per_bin)).astype(np.int32)
                bins_dev = torch.from_numpy(bins).cuda()
                want = np.stack([tables[g][x] for g, x in zip(bins, alphas)])
                for w in WAYS:                                            # warm-up: plans, scratch, attributes
                    run_calls(ctx, w, keys_dev, bins, bins_dev, prf, outs[:2], kind, want)
                res = {"%s_%s" % (w, m): [] for w in WAYS for m in ("host_ms", "per_call_ms", "launches_ms")}
                ok = True
                for _ in range(args.reps):
                    for w in WAYS:
                        h, d, dd, o = run_calls(ctx, w, keys_dev, bins, bins_dev, prf, outs, kind, want)
                        ok = ok and o
                        for m, v in zip(("host_ms", "per_call_ms", "launches_ms"), (h, d, dd)):
                            res["%s_%s" % (w, m)].append(v)
                row = {"kind": kind, "prf": NAMES[prf], "bins": nbins, "rows": n, "pairs": pairs, "E": e, "mix": mix,
                       "ok": bool(ok), **{k: statistics.median(v) for k, v in res.items()},
                       "plan_kernels_ms": plan_kernel_ms(ctx, keys_dev, bins, bins_dev, prf, outs)}
                rows.append(row)
                print(json.dumps(row), flush=True)
            del keys_dev, outs
        ctx.close()
    out = {"card": info, "reps": args.reps, "calls": args.calls, "rows": rows}
    path = args.out if os.path.isabs(args.out) else os.path.join(os.getcwd(), args.out)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("all ok" if all(r["ok"] for r in rows) else "CHECK FAILED")


if __name__ == "__main__":
    main()
