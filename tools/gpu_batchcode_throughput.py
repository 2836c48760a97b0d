"""Batch codes (b200dpf_batchcode_*): rows retrieved per second by queries of k wanted rows against k separate queries.

    python tools/gpu_batchcode_throughput.py [--reps 3] [--calls 5] [--out gpu_batchcode_throughput.json]

For n = 2^20 and 2^20 + 1 rows of 16 columns, every kind of key, AES and ChaCha20, and k = 8, 32, 128 wanted rows per
query with nbins = ceil(1.5 k), one process measures:
    batch_code  Q queries of k random rows (distinct within a query) on a batch-code context: the device plan and GPU
                keygen make compact queries (BatchCodeDPF.gen_queries_device), and one server evaluates them
                (b200dpf_group_eval_queries_device).  Rows retrieved = the placed wanted rows.
    separate    the same Q * k rows as Q * k keys of the kind on a plain trimmed context of the same table
                (b200dpf_eval_device), one key per wanted row.
Q * k = 4096 wanted rows per call.  "ms" is one server's evaluation (CUDA events around `calls` calls on one stream,
divided by `calls`; median of `reps` rounds, keys already on the device), and rows/s = retrieved rows / ms.  Both
ways' answers are checked once per case against the table with both servers' keys.
Also per case: the device planner's time for the Q queries (plan_ms, CUDA events, median), and per (n, kind, k) the
layout build: b200dpf_batchcode_create from a device table, wall clock around the call (context set-up included),
and as GB/s the bytes the scatter must move (n rows read, 3 n rows written) over that time.  "placed" is the
fraction of wanted rows the host planner places over 2,000 random queries (a host computation).  The card, its power
limit and SM clock are read in the same run (nvidia-smi, read-only queries).
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
import dpf  # noqa: E402

NAMES = {B.PRF_AES128: "AES128", B.PRF_CHACHA20: "CHACHA20"}
KINDS = {"std": ("", {}), "et": ("_et", {"early_termination": True}), "xor": ("_xor", {"xor": True})}
E = 16
WANTED_PER_CALL = 4096


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def timed(fn, calls, reps):
    """median over reps of (CUDA events around `calls` calls of fn) / calls, in ms; one warm-up call first"""
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(calls):
            fn()
        t1.record()
        t1.synchronize()
        out.append(t0.elapsed_time(t1) / calls)
    return statistics.median(out)


def rec(kind, a, b):
    return a ^ b if kind == "xor" else a - b


def distinct_rows(rng, n, nq, k):
    """nq queries of k distinct random rows"""
    rows = rng.randint(0, n, size=(nq, k)).astype(np.int64)
    for q in range(nq):
        while len(np.unique(rows[q])) < k:
            rows[q] = rng.randint(0, n, size=k)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default="gpu_batchcode_throughput.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU")
    out = {"card": card(), "entry_size": E, "wanted_rows_per_call": WANTED_PER_CALL, "rows": []}
    print(json.dumps({"card": out["card"]}), flush=True)
    rng = np.random.RandomState(1)
    for n in (1 << 20, (1 << 20) + 1):
        table = torch.randint(-2 ** 31, 2 ** 31, (n, E), dtype=torch.int64).to(torch.int32).cuda()
        table_h = table.cpu().numpy()
        for kname, (suffix, kw) in KINDS.items():
            plain = B.Context.__new__(B.Context)          # the separate queries' context: the same table, trimmed
            plain.n, plain.entry_size, plain.kind = n, E, suffix
            plain.handle = B.C.c_void_p()
            B._check(B.lib().b200dpf_create_trimmed(B.C.byref(plain.handle), B.C.c_void_p(table.data_ptr()), n, E, 0,
                                                    B.KIND_IDS[suffix]), "b200dpf_create_trimmed")
            for k in (8, 32, 128):
                nbins = (3 * k + 1) // 2
                nq = WANTED_PER_CALL // k
                d = dpf.BatchCodeDPF(B.PRF_AES128, 0, nbins, seed=k, **kw)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                d.eval_init(table)
                build_s = time.perf_counter() - t0
                placed = float((d.plan(distinct_rows(rng, n, 2000, k))[1] >= 0).float().mean())
                wanted = distinct_rows(rng, n, nq, k)
                wanted_dev = torch.as_tensor(wanted).cuda()
                alphas = torch.empty((nq, nbins), dtype=torch.int64, device="cuda")
                slots = torch.empty((nq, k), dtype=torch.int32, device="cuda")
                sdev = torch.cuda.current_stream().cuda_stream
                plan_ms = timed(lambda: dpf.dpf_cpp.batchcode_plan_device(wanted_dev.data_ptr(), nq, k, d.buffers,
                                                                          alphas.data_ptr(), slots.data_ptr(), sdev),
                                args.calls, args.reps)
                dom = B.trimmed_domain(n, suffix)
                sep_alphas = np.array([B.trimmed_alpha(int(r), n, suffix) for r in wanted.reshape(-1)], np.int64)
                ka = torch.empty((nq * k, B.KEY_WORDS), dtype=torch.int32, device="cuda")
                kb = torch.empty_like(ka)
                for prf in (B.PRF_AES128, B.PRF_CHACHA20):
                    d.prf_method = prf
                    qa, qb, sl = d.gen_queries_device(wanted_dev)
                    ra, rb = d.eval_queries_device(qa), d.eval_queries_device(qb)
                    rows, found = d.reconstruct(ra, rb, sl)
                    f = found.cpu().numpy()
                    assert np.array_equal(rows.cpu().numpy()[f], table_h[wanted[f]]), "batch code: wrong rows"
                    res = torch.empty((nq, nbins, E), dtype=torch.int32, device="cuda")
                    bc_ms = timed(lambda: d.eval_queries_device(qa, res), args.calls, args.reps)
                    retrieved = int(f.sum())
                    B._gen_batch_gpu(suffix, sep_alphas, dom, os.urandom(44 * nq * k), prf, 0,
                                     (ka.data_ptr(), kb.data_ptr()))
                    oa = torch.empty((nq * k, E), dtype=torch.int32, device="cuda")
                    ob = torch.empty_like(oa)
                    plain.eval_device(ka.data_ptr(), nq * k, prf, oa.data_ptr(), sdev)
                    plain.eval_device(kb.data_ptr(), nq * k, prf, ob.data_ptr(), sdev)
                    assert np.array_equal(rec(kname, oa, ob).cpu().numpy(), table_h[wanted.reshape(-1)]), "separate: wrong rows"
                    sep_ms = timed(lambda: plain.eval_device(ka.data_ptr(), nq * k, prf, oa.data_ptr(), sdev), args.calls,
                                   args.reps)
                    row = {"n": n, "kind": kname, "prf": NAMES[prf], "k": k, "nbins": nbins, "queries": nq,
                           "bin_rows_max": d.bin_sizes[0], "placed_host": round(placed, 5),
                           "placed_this_batch": retrieved / (nq * k),
                           "batch_code_ms": round(bc_ms, 4), "batch_code_rows_per_s": round(retrieved / bc_ms * 1e3),
                           "separate_ms": round(sep_ms, 4), "separate_rows_per_s": round(nq * k / sep_ms * 1e3),
                           "speedup": round((retrieved / bc_ms) / (nq * k / sep_ms), 3),
                           "plan_device_ms": round(plan_ms, 4), "layout_build_ms": round(build_s * 1e3, 2),
                           "layout_build_GBps": round(4 * n * E * 4 / build_s / 1e9, 2)}
                    out["rows"].append(row)
                    print(json.dumps(row), flush=True)
                d.close()
            plain.close()
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
