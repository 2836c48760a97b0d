"""DPFs/s of XOR-shared keys (128 rows per leaf) against standard and early-terminated keys, one process,
alternating.

    python tools/gpu_xor_throughput.py [--reps 3] [--iters 10] [--out gpu_xor_throughput.json]

For each shape the three kinds of context run in turn, `reps` rounds each, and every round times `iters`
evaluations of one batch of B keys with CUDA events (device-resident keys and result, after warm-up).
Every timed batch is checked: a - b = table[alpha] (standard, early-terminated) or a ^ b = table[alpha]
(XOR) for every key pair, and 4 keys bit-exact against the host evaluation.  The `s` sweep fixes the
work-item size of the XOR context only.  The card, its power limit and SM clock are read in the same run
(nvidia-smi).
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
import xor_oracle  # noqa: E402

NAMES = {B.PRF_AES128: "AES128", B.PRF_SALSA20: "SALSA20", B.PRF_CHACHA20: "CHACHA20"}
KINDS = ("std", "et", "xor")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "unavailable (%s)" % e
    return q


def make_keys(kind, n, batch, prf, seed):
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=batch).astype(np.int64)
    seeds = rng.randint(0, 256, size=44 * batch).astype(np.uint8).tobytes()
    gen = {"std": B.gen_batch_secure, "et": B.gen_batch_et, "xor": B.gen_batch_xor}[kind]
    a, b = gen(alphas, n, seeds, prf)
    return a, b, alphas


def host_result(kind, keys, prf, table):
    if kind == "xor":
        return xor_oracle.xor_rows(np.stack([xor_oracle.unpack_bits(B.eval_cpu_xor(k, prf)) for k in keys]), table)
    ev = B.eval_cpu_et if kind == "et" else B.eval_cpu
    return et_oracle.dot_u32(np.stack([ev(k, prf) for k in keys]), table)


def measure(ctx, kind, table, prf, batch, iters, seed):
    n, e = table.shape
    a, b, alphas = make_keys(kind, n, batch, prf, seed)
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
    ra, rb = out_a.cpu().numpy().view(np.uint32), out_b.cpu().numpy().view(np.uint32)
    rec = (ra ^ rb) if kind == "xor" else (ra - rb)
    ok = np.array_equal(rec.view(np.int32), table[alphas])
    ok = ok and np.array_equal(ra[:4].view(np.int32), host_result(kind, a[:4], prf, table))
    return ms, ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--quick", action="store_true", help="headline shape only")
    ap.add_argument("--part", choices=("all", "grid", "sweep"), default="all",
                    help="the grid of n, E and PRF, the s sweep, or both")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    shapes = [(B.PRF_AES128, 20, 16, 0)]
    if not args.quick:
        shapes = []
        if args.part != "sweep":
            shapes += [(prf, logn, e, 0) for e in (16, 128) for logn in (14, 16, 18, 20)
                       for prf in (B.PRF_AES128, B.PRF_SALSA20, B.PRF_CHACHA20)]
        if args.part != "grid":
            shapes += [(B.PRF_AES128, 20, 16, s) for s in (0, 1, 2, 3, 4, 5, 6)]     # 0: the automatic choice
            shapes += [(B.PRF_AES128, 16, 16, s) for s in (0, 1, 2, 3, 4, 5)]
    info = {"card": card(), "batch": args.batch, "rows": []}
    print("card:", info["card"], flush=True)
    tables = {}
    for prf, logn, e, s in shapes:
        key = (logn, e)
        if key not in tables:
            tables[key] = np.random.RandomState(logn * 1000 + e).randint(-2**31, 2**31, size=(1 << logn, e),
                                                                          dtype=np.int64).astype(np.int32)
        table = tables[key]
        ctxs = {"std": B.Context(table), "et": B.Context(table, early_termination=True), "xor": B.Context(table, xor=True)}
        if s:
            ctxs["xor"].set_option("subtree_log2", s)
        times = {k: [] for k in KINDS}
        ok = True
        for r in range(args.reps):
            for kind in KINDS:
                ms, good = measure(ctxs[kind], kind, table, prf, args.batch, args.iters, seed=r * 7 + logn)
                times[kind].append(ms)
                ok = ok and good
        for c in ctxs.values():
            c.close()
        med = {k: float(np.median(times[k])) for k in KINDS}
        row = {"prf": NAMES[prf], "n": 1 << logn, "E": e, "s_xor": s or "auto", "checked": ok}
        for k in KINDS:
            row[k + "_ms"] = med[k]
            row[k + "_dpfs"] = args.batch / med[k] * 1e3
            row[k + "_ms_all"] = times[k]
        row["xor_vs_et"] = med["et"] / med["xor"]
        row["xor_vs_std"] = med["std"] / med["xor"]
        info["rows"].append(row)
        print("%-8s n=2^%d E=%-3d s=%-4s std %8.3f ms  et %8.3f ms  xor %8.3f ms (%9.0f DPF/s)  xor/et x%.2f  xor/std x%.2f  %s"
              % (row["prf"], logn, e, row["s_xor"], med["std"], med["et"], med["xor"], row["xor_dpfs"], row["xor_vs_et"],
                 row["xor_vs_std"], "ok" if ok else "MISMATCH"), flush=True)
        if not ok:
            raise SystemExit("result check failed")
    info["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
