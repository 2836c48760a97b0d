"""Device time of trimmed contexts (any row count) against the same tables padded with zero rows to the next power
of two, one process, alternating.

    python tools/gpu_trimmed_throughput.py [--reps 3] [--iters 10] [--out gpu_trimmed_throughput.json]

Plain contexts: every kind, AES and ChaCha20, E = 16, B = 512, at n = 2^20 + 1, 1.5 * 2^20 and 2^21 - 2^14 (trimmed
against the padded table, which is what DPF(allow_non_pow2=True) uploads), and at n = 2^20 (trimmed against a plain
context: no padding to remove, so no change is expected).  Grouped query batches: 64 bins of 3,000 rows and 256 bins of
700 rows, 512 queries, AES, trimmed against the bins padded to 4,096 and 1,024 rows.

Every round times `iters` evaluations with CUDA events around device-resident keys and results, after a warm-up;
the contexts of a shape alternate round by round.  Every timed batch is checked: each key pair reconstructs its row
(a - b, or a ^ b for XOR-shared keys).  The card, its power limit and SM clock are read in the same run.
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
import plan_matrix  # noqa: E402

NAMES = {B.PRF_AES128: "AES128", B.PRF_CHACHA20: "CHACHA20"}
SUFFIX = {"standard": "", "et": "_et", "xor": "_xor"}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def plain_case(kind, prf, n, trimmed_vs_plain, reps, iters, batch=512, e=16):
    s = SUFFIX[kind]
    rng = np.random.RandomState(n)
    table = rng.randint(-2 ** 31, 2 ** 31, size=(n, e), dtype=np.int64).astype(np.int32)
    rows = rng.randint(0, n, size=batch).astype(np.int64)
    N = B.trimmed_domain(n, s)
    kw = dict(early_termination=kind == "et", xor=kind == "xor")
    trimmed = B.Context(table, trimmed=True, **kw)
    # the baseline: the table padded to N rows (allow_non_pow2), keys for the rows' own indices
    padded = np.zeros((N, e), np.int32)
    padded[:n] = table
    base = B.Context(padded, **kw)
    keys = {"trimmed": plan_matrix.gen_keys(kind, N, [B.trimmed_alpha(int(r), n, s) for r in rows], prf, 1),
            "padded": plan_matrix.gen_keys(kind, N, rows, prf, 1)}
    ctxs = {"trimmed": trimmed, "padded": base}
    out = {}
    for name, ctx in ctxs.items():
        ka, kb = (torch.from_numpy(k).cuda() for k in keys[name])
        oa, ob = (torch.zeros((batch, e), dtype=torch.int32, device="cuda") for _ in range(2))
        ctx.eval_device(ka.data_ptr(), batch, prf, oa.data_ptr())
        ctx.eval_device(kb.data_ptr(), batch, prf, ob.data_ptr())
        torch.cuda.synchronize()
        rec = plan_matrix.reconstruct(kind, oa.cpu().numpy(), ob.cpu().numpy())
        assert np.array_equal(rec, table[rows]), (kind, prf, n, name)
        out[name] = (ctx, ka, oa)
    ms = {name: [] for name in ctxs}
    for _ in range(reps):
        for name, (ctx, ka, oa) in out.items():
            ms[name].append(timed(lambda: ctx.eval_device(ka.data_ptr(), batch, prf, oa.data_ptr()), iters))
    res = {"kind": kind, "prf": NAMES[prf], "n": n, "domain": N, "table_rows": trimmed.table_rows,
           "baseline": "plain context" if trimmed_vs_plain else "padded to the domain",
           "ms_trimmed": ms["trimmed"], "ms_baseline": ms["padded"],
           "predicted_ratio": trimmed.table_rows / N}
    res["ratio"] = min(ms["trimmed"]) / min(ms["padded"])
    trimmed.close()
    base.close()
    return res


def group_case(nbins, rows_per_bin, reps, iters, nq=512, e=16, prf=B.PRF_AES128):
    rng = np.random.RandomState(nbins)
    tables = [rng.randint(-2 ** 31, 2 ** 31, size=(rows_per_bin, e), dtype=np.int64).astype(np.int32) for _ in range(nbins)]
    N = B.trimmed_domain(rows_per_bin)
    padded = [np.concatenate([t, np.zeros((N - rows_per_bin, e), np.int32)]) for t in tables]
    ctxs = {"trimmed": B.GroupContext(tables, trimmed=True), "padded": B.GroupContext(padded)}
    alphas = torch.from_numpy(rng.randint(0, rows_per_bin, size=(nq, nbins)).astype(np.int64)).cuda()
    seeds = torch.from_numpy(rng.randint(0, 256, size=(nq, nbins, 44)).astype(np.uint8)).cuda()
    ms, state = {}, {}
    for name, ctx in ctxs.items():
        qa = torch.zeros((nq, ctx.query_bytes), dtype=torch.uint8, device="cuda")
        qb = torch.zeros_like(qa)
        ctx.gen_queries_device(alphas.data_ptr(), seeds.data_ptr(), nq, prf, qa.data_ptr(), qb.data_ptr(), compact=True)
        oa = torch.zeros((nq, nbins, e), dtype=torch.int32, device="cuda")
        ob = torch.zeros_like(oa)
        ctx.eval_queries_device(qa.data_ptr(), nq, prf, oa.data_ptr(), compact=True)
        ctx.eval_queries_device(qb.data_ptr(), nq, prf, ob.data_ptr(), compact=True)
        torch.cuda.synchronize()
        rec = (oa.cpu().numpy().view(np.uint32) - ob.cpu().numpy().view(np.uint32)).view(np.int32)
        a = alphas.cpu().numpy()
        for g in range(nbins):
            assert np.array_equal(rec[:, g], tables[g][a[:, g]]), (name, g)
        state[name] = (ctx, qa, oa)
        ms[name] = []
    for _ in range(reps):
        for name, (ctx, qa, oa) in state.items():
            ms[name].append(timed(lambda: ctx.eval_queries_device(qa.data_ptr(), nq, prf, oa.data_ptr(), compact=True),
                                  iters))
    res = {"bins": nbins, "rows_per_bin": rows_per_bin, "queries": nq, "prf": NAMES[prf],
           "table_rows": ctxs["trimmed"].table_rows, "padded_rows": nbins * N,
           "ms_trimmed": ms["trimmed"], "ms_baseline": ms["padded"],
           "predicted_ratio": ctxs["trimmed"].table_rows / (nbins * N)}
    res["ratio"] = min(ms["trimmed"]) / min(ms["padded"])
    for ctx in ctxs.values():
        ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="gpu_trimmed_throughput.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gpu_trimmed_throughput: no CUDA device (this measures the GPU; there is nothing to fall back to)")
    results = {"card": card(), "plain": [], "grouped": []}
    print(results["card"], flush=True)
    for prf in (B.PRF_AES128, B.PRF_CHACHA20):
        for kind in ("standard", "et", "xor"):
            for n, vs_plain in (((1 << 20) + 1, False), (3 << 19, False), ((1 << 21) - (1 << 14), False), (1 << 20, True)):
                r = plain_case(kind, prf, n, vs_plain, args.reps, args.iters)
                results["plain"].append(r)
                print("%-8s %-8s n=%-8d rows=%-8d trimmed %.3f ms  %s %.3f ms  ratio %.3f (predicted %.3f)" % (
                    r["kind"], r["prf"], n, r["table_rows"], min(r["ms_trimmed"]), r["baseline"], min(r["ms_baseline"]),
                    r["ratio"], r["predicted_ratio"]), flush=True)
    for nbins, rows in ((64, 3000), (256, 700)):
        r = group_case(nbins, rows, args.reps, args.iters)
        results["grouped"].append(r)
        print("grouped %d x %d rows: trimmed %.3f ms  padded %.3f ms  ratio %.3f (predicted %.3f)" % (
            nbins, rows, min(r["ms_trimmed"]), min(r["ms_baseline"]), r["ratio"], r["predicted_ratio"]), flush=True)
    with open(args.out, "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
