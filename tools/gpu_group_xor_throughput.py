"""Batch-PIR throughput of XOR-shared keys on grouped contexts against standard and early-terminated keys on
grouped contexts and against XOR-shared keys bin by bin, one process, alternating.

    python tools/gpu_group_xor_throughput.py [--reps 3] [--iters 10] [--out gpu_group_xor_throughput.json]
                                             [--ab OTHER/libb200dpf.so]

Shapes are those of tools/gpu_group_et_throughput.py -- (bins, rows per bin, queries, columns), one key per
(query, bin), all pairs in one b200dpf_group_eval -- plus E = 128 at one shape.  For each shape and PRF four
ways of evaluating the batch run in turn, `reps` rounds each:
    std      a standard GroupContext                      (b200dpf_group_create)
    et       an early-terminated GroupContext             (b200dpf_group_create_et)
    xor      an XOR-shared GroupContext                   (b200dpf_group_create_xor)
    xor_bins one XOR-shared Context per bin, the device times of the bins summed (what a caller without
             grouped XOR evaluation does: one launch per bin and batch)
A round is the median device time (b200dpf_ctx_last_device_ms: the launches, copies excluded) of `iters`
evaluations after warm-up; the reported time is the median of the rounds.  Every timed batch is checked: the
two servers' results reconstruct table[bin][alpha] for every pair (a - b, or a ^ b), and two pairs per bin
are bit-exact against the host evaluation.  Then the work-item size s is swept at two shapes.  The card, its
power limit and SM clock are read in the same run (nvidia-smi).

--ab OTHER: instead, time the XOR-shared GroupContext of this build against one of the library at OTHER on
the same keys and tables, alternating (a scheduler A/B: OTHER is a build of other kernel code with the same
C ABI), every batch checked as above.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "tests")]
import b200dpf as B  # noqa: E402
import et_oracle  # noqa: E402
import xor_oracle  # noqa: E402

NAMES = {B.PRF_AES128: "AES128", B.PRF_CHACHA20: "CHACHA20"}
SHAPES = [(64, 12, 256, 16), (256, 10, 256, 16), (16, 14, 512, 16), (64, 12, 32, 16), (1024, 10, 64, 16),
          (64, 12, 256, 40), (16, 14, 512, 128)]
SWEEP_SHAPES = [(16, 14, 512, 16), (1024, 10, 64, 16)]
WAYS = ("std", "et", "xor", "xor_bins")
GEN = {"std": B.gen_batch_secure, "et": B.gen_batch_et, "xor": B.gen_batch_xor, "xor_bins": B.gen_batch_xor}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "unavailable (%s)" % e
    return q


def make_pairs(way, nbins, n, queries, prf, seed):
    """one key pair per (query, bin), query-major: pair q * nbins + g is for bin g"""
    rng = np.random.RandomState(seed)
    alphas = rng.randint(0, n, size=queries * nbins).astype(np.int64)
    seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
    a, b = GEN[way](alphas, n, seeds, prf)
    return a, b, np.tile(np.arange(nbins, dtype=np.int32), queries), alphas


def host_row(way, key, prf, table):
    if way in ("xor", "xor_bins"):
        return xor_oracle.xor_rows(xor_oracle.unpack_bits(B.eval_cpu_xor(key, prf)), table)[0]
    return et_oracle.dot_u32((B.eval_cpu_et if way == "et" else B.eval_cpu)(key, prf)[None, :], table)[0]


def check(way, tables, pairs, ra, rb, prf):
    a, _, bins, alphas = pairs
    if way in ("xor", "xor_bins"):
        rec = (ra.view(np.uint32) ^ rb.view(np.uint32)).view(np.int32)
    else:
        rec = (ra.view(np.uint32) - rb.view(np.uint32)).view(np.int32)
    ok = np.array_equal(rec, np.stack([tables[g][x] for g, x in zip(bins, alphas)]))
    for j in range(min(2 * len(tables), len(bins))):      # the first two queries: two pairs per bin
        ok = ok and np.array_equal(ra[j], host_row(way, a[j], prf, tables[bins[j]]))
    return ok


class Grouped:
    """a GroupContext of this build, or (lib != None) the same calls into another build of the library"""

    def __init__(self, tables, kind, lib=None):
        self.lib, self.e = lib, tables[0].shape[1]
        if lib is None:
            self.ctx = B.GroupContext(tables, early_termination=kind == "_et", xor=kind == "_xor")
            return
        lib.b200dpf_group_create_xor.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), B._i64p, C.c_int, C.c_int,
                                                 C.c_int]
        lib.b200dpf_group_eval.argtypes = [C.c_void_p, B._i32p, B._i32p, C.c_int64, C.c_int, B._i32p]
        lib.b200dpf_ctx_last_device_ms.argtypes = [C.c_void_p]
        lib.b200dpf_ctx_last_device_ms.restype = C.c_double
        lib.b200dpf_destroy.argtypes = [C.c_void_p]
        self.h = C.c_void_p()
        ptrs = (C.c_void_p * len(tables))(*[t.ctypes.data for t in tables])
        sizes = np.array([t.shape[0] for t in tables], np.int64)
        assert lib.b200dpf_group_create_xor(C.byref(self.h), ptrs, sizes, len(tables), self.e, 0) == 0

    def eval(self, keys, bins, prf):
        if self.lib is None:
            return self.ctx.eval(keys, bins, prf)
        out = np.zeros((len(keys), self.e), np.int32)
        assert self.lib.b200dpf_group_eval(self.h, keys, bins, len(keys), prf, out) == 0
        return out

    @property
    def last_device_ms(self):
        return self.ctx.last_device_ms if self.lib is None else self.lib.b200dpf_ctx_last_device_ms(self.h)

    def set_subtree_log2(self, s):
        self.ctx.set_subtree_log2(s)

    def close(self):
        if self.lib is None:
            self.ctx.close()
        else:
            self.lib.b200dpf_destroy(self.h)


class PerBin:
    """one XOR-shared Context per bin; a batch is one evaluation per bin, its device time the sum"""

    def __init__(self, tables):
        self.ctxs = [B.Context(t, xor=True) for t in tables]
        self.e = tables[0].shape[1]

    def eval(self, keys, bins, prf):
        out = np.zeros((len(keys), self.e), np.int32)
        self.ms = 0.0
        for g, ctx in enumerate(self.ctxs):
            sel = np.nonzero(bins == g)[0]
            out[sel] = ctx.eval(keys[sel], prf)
            self.ms += ctx.last_device_ms
        return out

    @property
    def last_device_ms(self):
        return self.ms

    def close(self):
        for c in self.ctxs:
            c.close()


def measure(ctx, way, tables, pairs, prf, iters):
    a, b, bins, _ = pairs
    for _ in range(2):                                   # warm-up
        ctx.eval(a, bins, prf)
    ms = []
    for _ in range(iters):
        ra = ctx.eval(a, bins, prf)
        ms.append(ctx.last_device_ms)
    rb = ctx.eval(b, bins, prf)
    return float(np.median(ms)), check(way, tables, pairs, ra, rb, prf)


def shape_tables(nbins, logn, e):
    n = 1 << logn
    return [np.random.RandomState(g * 7 + logn).randint(-2**31, 2**31, size=(n, e), dtype=np.int64).astype(np.int32)
            for g in range(nbins)]


def label(prf, nbins, logn, queries, e):
    return "%-8s %4d bins x 2^%d rows, %3d queries, E=%-3d" % (NAMES[prf], nbins, logn, queries, e)


def run_table(args, info):
    for nbins, logn, queries, e in SHAPES:
        tables = shape_tables(nbins, logn, e)
        ctxs = {"std": Grouped(tables, ""), "et": Grouped(tables, "_et"), "xor": Grouped(tables, "_xor"),
                "xor_bins": PerBin(tables)}
        for prf in (B.PRF_AES128, B.PRF_CHACHA20):
            pairs = {w: make_pairs(w, nbins, 1 << logn, queries, prf, seed=logn * 100 + nbins) for w in WAYS}
            times = {w: [] for w in WAYS}
            ok = True
            for _ in range(args.reps):
                for w in WAYS:
                    ms, good = measure(ctxs[w], w, tables, pairs[w], prf, args.iters)
                    times[w].append(ms)
                    ok = ok and good
            med = {w: float(np.median(times[w])) for w in WAYS}
            npairs = nbins * queries
            row = {"prf": NAMES[prf], "bins": nbins, "rows_per_bin": 1 << logn, "queries": queries, "pairs": npairs,
                   "E": e, "checked": ok}
            for w in WAYS:
                row[w + "_ms"] = med[w]
                row[w + "_ms_all"] = times[w]
                row[w + "_dpfs"] = npairs / med[w] * 1e3
            info["rows"].append(row)
            print("%s  std %7.3f  et %7.3f  xor %7.3f  xor bin by bin %8.3f ms   xor vs et x%.2f, vs bin by bin x%.2f  %s"
                  % (label(prf, nbins, logn, queries, e), med["std"], med["et"], med["xor"], med["xor_bins"],
                     med["et"] / med["xor"], med["xor_bins"] / med["xor"], "ok" if ok else "MISMATCH"), flush=True)
            if not ok:
                raise SystemExit("result check failed")
        for c in ctxs.values():
            c.close()


def run_sweep(args, info):
    for nbins, logn, queries, e in SWEEP_SHAPES:
        tables = shape_tables(nbins, logn, e)
        ctx = Grouped(tables, "_xor")
        for prf in (B.PRF_AES128, B.PRF_CHACHA20):
            pairs = make_pairs("xor", nbins, 1 << logn, queries, prf, seed=logn * 100 + nbins)
            svals = [0] + list(range(1, min(logn - 7, 6) + 1))
            times = {s: [] for s in svals}
            ok = True
            for _ in range(args.reps):
                for s in svals:
                    ctx.set_subtree_log2(s)
                    ms, good = measure(ctx, "xor", tables, pairs, prf, args.iters)
                    times[s].append(ms)
                    ok = ok and good
            ctx.set_subtree_log2(0)
            med = {s: float(np.median(times[s])) for s in svals}
            info["sweep"].append({"prf": NAMES[prf], "bins": nbins, "rows_per_bin": 1 << logn, "queries": queries, "E": e,
                                  "ms_by_s": {("auto" if s == 0 else str(s)): med[s] for s in svals}, "checked": ok})
            print("%s  s sweep: %s  %s" % (label(prf, nbins, logn, queries, e),
                                           "  ".join("%s %.3f" % ("auto" if s == 0 else "s=%d" % s, med[s]) for s in svals),
                                           "ok" if ok else "MISMATCH"), flush=True)
            if not ok:
                raise SystemExit("result check failed")
        ctx.close()


def run_ab(args, info):
    other = C.CDLL(os.path.abspath(args.ab))
    for nbins, logn, queries, e in SHAPES[:6]:
        tables = shape_tables(nbins, logn, e)
        ctxs = {"this": Grouped(tables, "_xor"), "other": Grouped(tables, "_xor", lib=other)}
        for prf in (B.PRF_AES128, B.PRF_CHACHA20):
            pairs = make_pairs("xor", nbins, 1 << logn, queries, prf, seed=logn * 100 + nbins)
            times = {k: [] for k in ctxs}
            ok = True
            for _ in range(args.reps):
                for k, ctx in ctxs.items():
                    ms, good = measure(ctx, "xor", tables, pairs, prf, args.iters)
                    times[k].append(ms)
                    ok = ok and good
            med = {k: float(np.median(v)) for k, v in times.items()}
            info["ab"].append({"prf": NAMES[prf], "bins": nbins, "rows_per_bin": 1 << logn, "queries": queries, "E": e,
                               "this_ms": med["this"], "other_ms": med["other"], "this_ms_all": times["this"],
                               "other_ms_all": times["other"], "checked": ok})
            print("%s  this build %7.3f ms  other build %7.3f ms  x%.2f  %s"
                  % (label(prf, nbins, logn, queries, e), med["this"], med["other"], med["other"] / med["this"],
                     "ok" if ok else "MISMATCH"), flush=True)
            if not ok:
                raise SystemExit("result check failed")
        for c in ctxs.values():
            c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--ab", default=None, help="libb200dpf.so of another build: scheduler A/B only")
    args = ap.parse_args()
    info = {"card": card(), "rows": [], "sweep": [], "ab": []}
    print("card:", info["card"], flush=True)
    if args.ab:
        run_ab(args, info)
    else:
        run_table(args, info)
        run_sweep(args, info)
    info["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
