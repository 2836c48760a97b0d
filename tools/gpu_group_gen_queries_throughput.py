"""Batch-PIR query generation on the GPU (b200dpf_group_gen_queries_device) against the host's keygen and
pack_queries, and against the evaluation of the same batch (b200dpf_group_eval_queries_device).

    python tools/gpu_group_gen_queries_throughput.py [--reps 3] [--calls 20] [--out gpu_group_gen_queries_throughput.json]

Shapes are (bins, log2 rows per bin, queries, columns), one key pair per (query, bin): those of DESIGN.md section
8's query table.  XOR-shared and early-terminated keys run every shape, standard keys two, each with AES and
ChaCha20.  Per shape, kind and PRF, in each of `reps` alternating rounds:
    gen wire / gen compact  `calls` generator calls back to back on one stream (both servers' queries per call),
                            CUDA events around all of them divided by `calls`
    host gen                gen_batch<kind> of both servers' keys on all host cores (one call: every bin of a
                            shape has the same size), wall clock
    host pack               GroupContext.pack_queries of both servers' keys, wall clock
    eval                    `calls` b200dpf_group_eval_queries_device calls on compact queries (one server's batch
                            each), CUDA events per call
    loop / eval alone       `calls` iterations on one stream of: generate fresh compact queries (new rows and seeds
                            per iteration, made on the device beforehand) and evaluate both servers' batches; and the
                            same two evaluations per iteration without the generator.  CUDA events per iteration.
Reported times are medians of the rounds.  Every timed batch is checked: the generator's last outputs of each way
are evaluated and reconstruct table[bin][alpha] (a - b, or a ^ b), and every iteration of the loop reconstructs
its own rows.  The card, its power limit and SM clock are read in the same run (nvidia-smi, read-only queries).
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


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unavailable (%s)" % e


def reconstructs(kind, ra, rb, want):
    ra, rb = ra.reshape(want.shape), rb.reshape(want.shape)
    if kind == "xor":
        return np.array_equal((ra.view(np.uint32) ^ rb.view(np.uint32)).view(np.int32), want)
    return np.array_equal((ra.view(np.uint32) - rb.view(np.uint32)).view(np.int32), want)


def selected(tables, alphas):
    return np.stack([np.stack([tables[g][x] for g, x in enumerate(row)]) for row in alphas])


def timed(stream, calls, body):
    """CUDA events around `calls` runs of body(i) on `stream`, per run (ms)"""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(calls):
        body(i)
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default="gpu_group_gen_queries_throughput.json")
    args = ap.parse_args()
    info = card()
    print("card:", info, "host cores:", os.cpu_count(), flush=True)
    rows = []
    cases = [(k, sh) for sh in SHAPES for k in ("xor", "et")] + [("std", sh) for sh in STD_SHAPES]
    dev = torch.device("cuda", 0)
    for kind, (nbins, lg, queries, e) in cases:
        n = 1 << lg
        tables = [np.random.RandomState(1000 + g).randint(-2**31, 2**31, size=(n, e), dtype=np.int64).astype(np.int32)
                  for g in range(nbins)]
        ctx = B.GroupContext(tables, **KINDS[kind][1])
        qb = ctx.query_bytes
        pairs = queries * nbins
        st = torch.cuda.Stream(dev)
        gen = torch.Generator(device=dev).manual_seed(nbins + lg)
        with torch.cuda.stream(st):
            # `calls` fresh batches of rows and seeds for the loop; batch 0 also feeds the other ways
            alphas = [torch.randint(0, n, (queries, nbins), dtype=torch.int64, device=dev, generator=gen)
                      for _ in range(args.calls)]
            seeds = [torch.randint(0, 256, (queries, nbins, 44), dtype=torch.uint8, device=dev, generator=gen)
                     for _ in range(args.calls)]
            wire = [torch.empty((queries, nbins, B.KEY_WORDS), dtype=torch.int32, device=dev) for _ in range(2)]
            comp = [torch.empty((queries, qb), dtype=torch.uint8, device=dev) for _ in range(2)]
            loopq = [[torch.empty((queries, qb), dtype=torch.uint8, device=dev) for _ in range(2)] for _ in range(args.calls)]
            outs = [[torch.empty((queries, nbins, e), dtype=torch.int32, device=dev) for _ in range(2)] for _ in range(args.calls)]
        st.synchronize()
        al_host = [a.cpu().numpy() for a in alphas]
        want = [selected(tables, a) for a in al_host]
        seeds0 = seeds[0].cpu().numpy()
        for prf in (B.PRF_AES128, B.PRF_CHACHA20):
            def gen_into(i, dst, compact, j=0):
                ctx.gen_queries_device(alphas[j].data_ptr(), seeds[j].data_ptr(), queries, prf, dst[0].data_ptr(),
                                       dst[1].data_ptr(), st.cuda_stream, compact=compact)

            def ev(q, o, compact=True):
                ctx.eval_queries_device(q.data_ptr(), queries, prf, o.data_ptr(), st.cuda_stream, compact=compact)

            def loop_body(i):
                gen_into(i, loopq[i], True, j=i)
                ev(loopq[i][0], outs[i][0])
                ev(loopq[i][1], outs[i][1])

            def eval_pair(i):
                ev(comp[0], outs[i][0])
                ev(comp[1], outs[i][1])

            # warm-up: every way, both formats planned
            gen_into(0, wire, False)
            gen_into(0, comp, True)
            ev(wire[0], outs[0][0], compact=False)
            loop_body(0)
            eval_pair(0)
            st.synchronize()
            res = {k: [] for k in ("gen_wire_ms", "gen_compact_ms", "host_gen_ms", "host_pack_ms", "eval_ms", "loop_ms",
                                   "eval_alone_ms")}
            ok = True
            for _ in range(args.reps):
                res["gen_wire_ms"].append(timed(st, args.calls, lambda i: gen_into(i, wire, False)))
                res["gen_compact_ms"].append(timed(st, args.calls, lambda i: gen_into(i, comp, True)))
                ev(wire[0], outs[0][0], compact=False)
                ev(wire[1], outs[0][1], compact=False)
                st.synchronize()
                ok = ok and reconstructs(kind, outs[0][0].cpu().numpy(), outs[0][1].cpu().numpy(), want[0])
                res["eval_ms"].append(timed(st, args.calls, lambda i: ev(comp[i % 2], outs[i][i % 2])))
                for i in range(0, args.calls - 1, 2):
                    ok = ok and reconstructs(kind, outs[i][0].cpu().numpy(), outs[i + 1][1].cpu().numpy(), want[0])
                res["loop_ms"].append(timed(st, args.calls, loop_body))
                ok = ok and all(reconstructs(kind, outs[i][0].cpu().numpy(), outs[i][1].cpu().numpy(), want[i])
                                for i in range(args.calls))
                res["eval_alone_ms"].append(timed(st, args.calls, eval_pair))
                ok = ok and all(reconstructs(kind, outs[i][0].cpu().numpy(), outs[i][1].cpu().numpy(), want[0])
                                for i in range(args.calls))
                t0 = time.perf_counter()            # every bin has n rows: one batch of all pairs, query-major
                ka, kb = KINDS[kind][0](al_host[0].reshape(-1), n, seeds0.tobytes(), prf)
                res["host_gen_ms"].append((time.perf_counter() - t0) * 1e3)
                ka, kb = ka.reshape(queries, nbins, B.KEY_WORDS), kb.reshape(queries, nbins, B.KEY_WORDS)
                t0 = time.perf_counter()
                packed = [ctx.pack_queries(ka), ctx.pack_queries(kb)]
                res["host_pack_ms"].append((time.perf_counter() - t0) * 1e3)
                ok = ok and all(np.array_equal(p, c.cpu().numpy()) for p, c in zip(packed, comp))
            row = {"kind": kind, "prf": NAMES[prf], "bins": nbins, "rows": n, "queries": queries, "E": e, "pairs": pairs,
                   "ok": bool(ok), **{k: statistics.median(v) for k, v in res.items()}}
            row["keeps_up"] = row["gen_compact_ms"] <= row["eval_ms"]
            rows.append(row)
            print(json.dumps(row), flush=True)
        ctx.close()
        del alphas, seeds, wire, comp, loopq, outs
    out = {"card": info, "host_cores": os.cpu_count(), "reps": args.reps, "calls": args.calls, "rows": rows}
    path = args.out if os.path.isabs(args.out) else os.path.join(os.getcwd(), args.out)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("all ok" if all(r["ok"] for r in rows) else "CHECK FAILED")


if __name__ == "__main__":
    main()
