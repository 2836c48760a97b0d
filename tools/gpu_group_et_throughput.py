"""Batch-PIR throughput of early-terminated keys against standard keys on grouped contexts, one process,
alternating.

    python tools/gpu_group_et_throughput.py [--reps 3] [--iters 10] [--out gpu_group_et_throughput.json]

Shapes are those of tools/gpu_batch_pir.py -- (bins, rows per bin, queries), one key per (query, bin), all
pairs in one b200dpf_group_eval -- at 16 columns, plus one 40-column line.  For each shape and PRF a
standard and an early-terminated GroupContext hold the same tables; they run in turn, `reps` rounds each,
and a round is the median device time (b200dpf_ctx_last_device_ms: the launches, copies excluded) of
`iters` evaluations after warm-up.  The reported time is the median of the rounds.  Every timed batch is
checked: a - b = table[bin][alpha] for every pair, and two pairs per bin bit-exact against the host
evaluation.  The card, its power limit and SM clock are read in the same run (nvidia-smi).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "tests")]
import b200dpf as B  # noqa: E402
import et_oracle  # noqa: E402

NAMES = {B.PRF_AES128: "AES128", B.PRF_CHACHA20: "CHACHA20"}
SHAPES = [(64, 12, 256, 16), (256, 10, 256, 16), (16, 14, 512, 16), (64, 12, 32, 16), (1024, 10, 64, 16),
          (64, 12, 256, 40)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "unavailable (%s)" % e
    return q


def make_pairs(et, nbins, n, queries, prf, seed):
    """one key pair per (query, bin), query-major: pair q * nbins + g is for bin g"""
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=queries * nbins).astype(np.int64)
    seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
    a, b = (B.gen_batch_et if et else B.gen_batch_secure)(alphas, n, seeds, prf)
    return a, b, np.tile(np.arange(nbins, dtype=np.int32), queries), alphas


def measure(ctx, et, tables, pairs, prf, iters):
    a, b, bins, alphas = pairs
    for _ in range(2):                                   # warm-up
        ctx.eval(a, bins, prf)
    ms = []
    for _ in range(iters):
        ra = ctx.eval(a, bins, prf)
        ms.append(ctx.last_device_ms)
    rb = ctx.eval(b, bins, prf)
    ok = np.array_equal((ra.view(np.uint32) - rb.view(np.uint32)).view(np.int32),
                        np.stack([tables[g][x] for g, x in zip(bins, alphas)]))
    host = B.eval_cpu_et if et else B.eval_cpu
    nbins = len(tables)
    for j in list(range(nbins)) + list(range(nbins, 2 * nbins)):   # the first two queries: two pairs per bin
        if j < len(bins):
            ok = ok and np.array_equal(ra[j], et_oracle.dot_u32(host(a[j], prf)[None, :], tables[bins[j]])[0])
    return float(np.median(ms)), ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    info = {"card": card(), "rows": []}
    print("card:", info["card"], flush=True)
    for nbins, logn, queries, e in SHAPES:
        n = 1 << logn
        tables = [np.random.RandomState(g * 7 + logn).randint(-2**31, 2**31, size=(n, e), dtype=np.int64).astype(np.int32)
                  for g in range(nbins)]
        ctxs = {False: B.GroupContext(tables), True: B.GroupContext(tables, early_termination=True)}
        for prf in (B.PRF_AES128, B.PRF_CHACHA20):
            pairs = {et: make_pairs(et, nbins, n, queries, prf, seed=logn * 100 + nbins) for et in (False, True)}
            times = {False: [], True: []}
            ok = True
            for _ in range(args.reps):
                for et in (False, True):
                    ms, good = measure(ctxs[et], et, tables, pairs[et], prf, args.iters)
                    times[et].append(ms)
                    ok = ok and good
            std, et = float(np.median(times[False])), float(np.median(times[True]))
            npairs = nbins * queries
            row = {"prf": NAMES[prf], "bins": nbins, "rows_per_bin": n, "queries": queries, "pairs": npairs, "E": e,
                   "std_ms": std, "et_ms": et, "std_dpfs": npairs / std * 1e3, "et_dpfs": npairs / et * 1e3,
                   "speedup": std / et, "std_ms_all": times[False], "et_ms_all": times[True], "checked": ok}
            info["rows"].append(row)
            print("%-8s %4d bins x 2^%d rows, %3d queries, E=%-2d  std %8.3f ms (%10.0f DPF/s)  et %8.3f ms (%10.0f DPF/s)"
                  "  x%.2f  %s" % (row["prf"], nbins, logn, queries, e, std, row["std_dpfs"], et, row["et_dpfs"],
                                   row["speedup"], "ok" if ok else "MISMATCH"), flush=True)
            if not ok:
                raise SystemExit("result check failed")
        for c in ctxs.values():
            c.close()
    info["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
