"""Create time: b200dpf_create and b200dpf_group_create by wall clock, for one or more builds of libb200dpf.so in one
process, alternated round by round.

    python tools/gpu_create_time.py [--lib A/libb200dpf.so --lib B/libb200dpf.so] [--reps 7] [--out gpu_create_time.json]

plain    n = 2^20 and 2^24, E = 16, the whole table and shard 0 of 4, from a pageable host table (numpy) and a device
         table (a CUDA tensor on the context's device)
grouped  64 bins of n / 64 rows each (n = 2^20 and 2^24), E = 16, from host and from device
Each figure is the wall clock of one create call, which returns once the table is on the device; destroy is not
timed.  Every (build, shape) runs once before the timed rounds.  Rounds alternate the builds in turn, and the line
gives the median, the minimum and the maximum over `reps` rounds.  With no --lib the build next to this tree is
timed alone.  The card, its power limit and SM clock are read in the same run (nvidia-smi, read-only queries).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E = 16
BINS = 64


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def load(path):
    lib = C.CDLL(os.path.abspath(path))
    lib.b200dpf_create.argtypes = [C.POINTER(C.c_void_p), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.b200dpf_group_create.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int, C.c_int,
                                         C.c_int]
    lib.b200dpf_destroy.argtypes = [C.c_void_p]
    return lib


def create_ms(lib, shape, src):
    """wall clock of one create of `shape` from the table at address src, in ms"""
    kind, n, shards = shape
    h = C.c_void_p()
    if kind == "plain":
        t0 = time.perf_counter()
        rc = lib.b200dpf_create(C.byref(h), C.c_void_p(src), n, E, 0, 0, shards)
    else:
        rows = n // BINS
        ptrs = (C.c_void_p * BINS)(*[src + g * rows * E * 4 for g in range(BINS)])
        sizes = (C.c_int64 * BINS)(*[rows] * BINS)
        t0 = time.perf_counter()
        rc = lib.b200dpf_group_create(C.byref(h), ptrs, sizes, BINS, E, 0)
    ms = (time.perf_counter() - t0) * 1e3
    if rc:
        raise RuntimeError("create %s failed (%d)" % (shape, rc))
    lib.b200dpf_destroy(h)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", help="a libb200dpf.so to time (repeatable; default: this tree's)")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default="gpu_create_time.json")
    args = ap.parse_args()
    libs = args.lib or [os.path.join(ROOT, "gpu-dpf_b200", "libb200dpf.so")]
    loaded = [load(p) for p in libs]
    print("card:", card())
    shapes = [(kind, n, shards) for n in (1 << 20, 1 << 24) for kind, shards in (("plain", 1), ("plain", 4), ("grouped", 1))]
    rng = np.random.default_rng(1)
    results = []
    for n in (1 << 20, 1 << 24):
        host = rng.integers(0, 2**32, size=(n, E), dtype=np.uint32).view(np.int32)
        dev = torch.from_numpy(host).cuda()
        torch.cuda.synchronize()
        for shape in (s for s in shapes if s[1] == n):
            for where, src in (("host", host.ctypes.data), ("device", dev.data_ptr())):
                for lib in loaded:
                    create_ms(lib, shape, src)
                times = [[] for _ in libs]
                for _ in range(args.reps):
                    for i, lib in enumerate(loaded):
                        times[i].append(create_ms(lib, shape, src))
                for path, t in zip(libs, times):
                    row = {"lib": path, "kind": shape[0], "n": n, "shards": shape[2], "source": where,
                           "median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t), "ms": t}
                    results.append(row)
                    print("%-8s n=2^%d shards=%d %-6s %-50s median %8.2f ms  [%8.2f, %8.2f]" % (
                        shape[0], n.bit_length() - 1, shape[2], where, path[-50:], row["median_ms"], row["min_ms"],
                        row["max_ms"]), flush=True)
        del dev
        torch.cuda.empty_cache()
    with open(args.out, "w") as f:
        json.dump({"card": card(), "E": E, "bins": BINS, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
