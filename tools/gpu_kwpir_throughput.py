"""Keyword PIR (b200dpf_kwpir_*): the layout build, and one server's query time against an index query of the same items.

    python tools/gpu_kwpir_throughput.py [--reps 3] [--calls 5] [--out gpu_kwpir_throughput.json]

build   n = 2^20 and 2^24 distinct random keywords, value sizes E = 14 and 30, m = ceil(1.3 n / 3), keywords and values
        in host memory (numpy) or on the device (CUDA tensors): b200dpf_kwpir_create's wall clock (context set-up, the
        duplicate check, the placement, the row scatter and the host-to-device copies included), and the placement
        rounds alone by CUDA events with the rounds taken (b200dpf_kwpir_build_stats).  Standard keys: the kind does
        not enter the build.
query   n = 2^20 items, E = 14 and 16, every kind of key, AES and ChaCha20: 512 compact queries of present keywords made on
        the GPU (KeywordDPF.gen_queries_device) and evaluated by one server (b200dpf_group_eval_queries_device, three
        bins of m rows and E + 2 columns), against 512 keys of the kind on a plain trimmed context of the same n rows of
        E columns queried by index (b200dpf_eval_device).  "ms" is CUDA events around `calls` calls on one stream,
        divided by `calls`, median of `reps` rounds, keys already on the device.  Every timed batch is reconstructed
        with both servers' keys and checked against the values.
The card, its power limit and SM clock are read in the same run (nvidia-smi, read-only queries).
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
QUERIES = 512


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


def keywords(n, salt):
    """n distinct keywords: the SplitMix64 finalizer (a bijection) of 0..n-1 xor a salt, 2^64 - 1 excluded"""
    z = np.arange(n + 1, dtype=np.uint64) ^ np.uint64(salt)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
    z = z ^ (z >> np.uint64(31))
    return z[z != np.uint64((1 << 64) - 1)][:n]


def build(n, e, on_device, kw, values):
    m = -(-13 * n // 30)
    if on_device:
        kt = torch.as_tensor(kw.view(np.int64)).cuda()
        vt = torch.as_tensor(values).cuda()
        kp, vp = B.C.c_void_p(kt.data_ptr()), B.C.c_void_p(vt.data_ptr())
    else:
        kp, vp = kw.ctypes.data_as(B.C.c_void_p), values.ctypes.data_as(B.C.c_void_p)
    ctx = B.KeywordContext.__new__(B.KeywordContext)
    ctx.n, ctx.value_size, ctx.entry_size, ctx.kind, ctx._trimmed = n, e, e + 2, "", True
    ctx.handle = B.C.c_void_p()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    B._check(B.lib().b200dpf_kwpir_create(B.C.byref(ctx.handle), kp, vp, n, e, m, 1, 0, 0), "b200dpf_kwpir_create")
    wall = time.perf_counter() - t0
    rounds, place_ms = ctx.build_stats
    ctx.close()
    return {"n": n, "value_size": e, "m": m, "inputs": "device" if on_device else "host", "create_ms": round(wall * 1e3, 2),
            "rounds": rounds, "placement_ms": round(place_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default="gpu_kwpir_throughput.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU")
    out = {"card": card(), "queries": QUERIES, "build": [], "query": []}
    print(json.dumps({"card": out["card"]}), flush=True)
    rng = np.random.RandomState(1)
    for n in (1 << 20, 1 << 24):
        kw = keywords(n, 0x1234)
        for e in (14, 30):
            values = rng.randint(-2 ** 31, 2 ** 31, size=(n, e), dtype=np.int64).astype(np.int32)
            for on_device in (False, True):
                row = build(n, e, on_device, kw, values)
                out["build"].append(row)
                print(json.dumps(row), flush=True)
    n = 1 << 20
    kw = keywords(n, 0x5678)
    sdev = torch.cuda.current_stream().cuda_stream
    for e in (14, 16):
        values = rng.randint(-2 ** 31, 2 ** 31, size=(n, e), dtype=np.int64).astype(np.int32)
        vt = torch.as_tensor(values).cuda()
        pick = rng.choice(n, QUERIES, replace=False)
        qkw = torch.as_tensor(kw[pick].view(np.int64)).cuda()
        for kname, (suffix, kwargs) in KINDS.items():
            d = dpf.KeywordDPF(B.PRF_AES128, 0, seed=7, **kwargs)
            d.eval_init(kw, values)
            plain = B.Context.__new__(B.Context)      # the index queries' context: the same n values, trimmed
            plain.n, plain.entry_size, plain.kind = n, e, suffix
            plain.handle = B.C.c_void_p()
            B._check(B.lib().b200dpf_create_trimmed(B.C.byref(plain.handle), B.C.c_void_p(vt.data_ptr()), n, e, 0,
                                                    B.KIND_IDS[suffix]), "b200dpf_create_trimmed")
            dom = B.trimmed_domain(n, suffix)
            idx_alphas = np.array([B.trimmed_alpha(int(r), n, suffix) for r in pick], np.int64)
            ka = torch.empty((QUERIES, B.KEY_WORDS), dtype=torch.int32, device="cuda")
            kb = torch.empty_like(ka)
            for prf in (B.PRF_AES128, B.PRF_CHACHA20):
                d.prf_method = prf
                qa, qb = d.gen_queries_device(qkw)
                res_a = torch.empty((QUERIES, 3, e + 2), dtype=torch.int32, device="cuda")
                res_b = torch.empty_like(res_a)
                kw_ms = timed(lambda: d.eval_queries_device(qa, res_a), args.calls, args.reps)
                d.eval_queries_device(qb, res_b)
                vals, found = d.reconstruct(res_a, res_b, qkw)
                assert bool(found.all()) and np.array_equal(vals.cpu().numpy(), values[pick]), "keyword: wrong values"
                B._gen_batch_gpu(suffix, idx_alphas, dom, os.urandom(44 * QUERIES), prf, 0, (ka.data_ptr(), kb.data_ptr()))
                oa = torch.empty((QUERIES, e), dtype=torch.int32, device="cuda")
                ob = torch.empty_like(oa)
                idx_ms = timed(lambda: plain.eval_device(ka.data_ptr(), QUERIES, prf, oa.data_ptr(), sdev), args.calls, args.reps)
                plain.eval_device(kb.data_ptr(), QUERIES, prf, ob.data_ptr(), sdev)
                r = oa ^ ob if kname == "xor" else oa - ob
                assert np.array_equal(r.cpu().numpy(), values[pick]), "index: wrong rows"
                row = {"n": n, "value_size": e, "columns": e + 2, "m": d.m, "kind": kname, "prf": NAMES[prf],
                       "keyword_ms": round(kw_ms, 4), "index_ms": round(idx_ms, 4), "ratio": round(kw_ms / idx_ms, 3),
                       "rows_ratio": round(3 * d.m / n, 3)}
                out["query"].append(row)
                print(json.dumps(row), flush=True)
            plain.close()
            d.close()
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
