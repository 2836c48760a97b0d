"""DPFs/s of early-terminated keys (four rows per leaf) against standard keys, one process, alternating.

    python tools/gpu_et_throughput.py [--reps 3] [--iters 10] [--out gpu_et_throughput.json]

For each shape the two kinds of context run in turn, `reps` rounds each, and every round times `iters`
evaluations of one batch of B keys with CUDA events (device-resident keys and result, after warm-up).
Every timed batch is checked: a - b = table[alpha] for every key pair, and 4 keys bit-exact against
the host evaluation.  The card, its power limit and SM clock are read in the same run (nvidia-smi).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "tests")]
import b200dpf as B  # noqa: E402
import et_oracle  # noqa: E402

NAMES = {B.PRF_AES128: "AES128", B.PRF_SALSA20: "SALSA20", B.PRF_CHACHA20: "CHACHA20"}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "unavailable (%s)" % e
    return q


def make_keys(et, n, batch, prf, seed):
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=batch).astype(np.int64)
    seeds = rng.randint(0, 256, size=44 * batch).astype(np.uint8).tobytes()
    gen = B.gen_batch_et if et else B.gen_batch_secure
    a, b = gen(alphas, n, seeds, prf)
    return a, b, alphas


def host_shares(et, key, prf):
    return B.eval_cpu_et(key, prf) if et else B.eval_cpu(key, prf)


def measure(ctx, et, table, prf, batch, iters, seed, s=0):
    n, e = table.shape
    a, b, alphas = make_keys(et, n, batch, prf, seed)
    if s:
        ctx.set_option("subtree_log2", s)
    ka, kb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    out_a = torch.zeros((batch, e), dtype=torch.int32, device="cuda")
    out_b = torch.zeros_like(out_a)
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(3):                                   # warm-up
        ctx.eval_device(ka.data_ptr(), batch, prf, out_a.data_ptr(), stream)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        ctx.eval_device(ka.data_ptr(), batch, prf, out_a.data_ptr(), stream)
    t1.record()
    t1.synchronize()
    ms = t0.elapsed_time(t1) / iters
    ctx.eval_device(kb.data_ptr(), batch, prf, out_b.data_ptr(), stream)
    torch.cuda.synchronize()
    ra, rb = out_a.cpu().numpy(), out_b.cpu().numpy()
    ok = np.array_equal((ra.view(np.uint32) - rb.view(np.uint32)).view(np.int32), table[alphas])
    want = et_oracle.dot_u32(np.stack([host_shares(et, k, prf) for k in a[:4]]), table)
    ok = ok and np.array_equal(ra[:4], want)
    return ms, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--quick", action="store_true", help="headline shape only")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    shapes = [(B.PRF_AES128, 20, 16, 0)]
    if not args.quick:
        shapes = [(prf, logn, 16, 0) for logn in (14, 16, 18, 20) for prf in (B.PRF_AES128, B.PRF_SALSA20, B.PRF_CHACHA20)]
        shapes += [(B.PRF_AES128, 20, 128, 0)] + [(B.PRF_AES128, 20, 16, s) for s in (3, 4, 5, 6, 7, 8)]
    info = {"card": card(), "batch": args.batch, "rows": []}
    print("card:", info["card"], flush=True)
    tables = {}
    for prf, logn, e, s in shapes:
        key = (logn, e)
        if key not in tables:
            tables[key] = np.random.RandomState(logn * 1000 + e).randint(-2**31, 2**31, size=(1 << logn, e),
                                                                          dtype=np.int64).astype(np.int32)
        table = tables[key]
        ctxs = {False: B.Context(table), True: B.Context(table, early_termination=True)}
        times = {False: [], True: []}
        ok = True
        for r in range(args.reps):
            for et in (False, True):
                ms, good = measure(ctxs[et], et, table, prf, args.batch, args.iters, seed=r * 7 + logn, s=s)
                times[et].append(ms)
                ok = ok and good
        for c in ctxs.values():
            c.close()
        std, et = float(np.median(times[False])), float(np.median(times[True]))
        row = {"prf": NAMES[prf], "n": 1 << logn, "E": e, "s": s or "auto", "std_ms": std, "et_ms": et,
               "std_dpfs": args.batch / std * 1e3, "et_dpfs": args.batch / et * 1e3, "speedup": std / et,
               "std_ms_all": times[False], "et_ms_all": times[True], "checked": ok}
        info["rows"].append(row)
        print("%-8s n=2^%d E=%-3d s=%-4s std %8.3f ms (%9.0f DPF/s)  et %8.3f ms (%9.0f DPF/s)  x%.2f  %s"
              % (row["prf"], logn, e, row["s"], std, row["std_dpfs"], et, row["et_dpfs"], row["speedup"],
                 "ok" if ok else "MISMATCH"), flush=True)
        if not ok:
            raise SystemExit("result check failed")
    info["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
