"""Cost of row updates on a live context (b200dpf_update_rows / _update_rows_device) against rebuilding it.

At n = 2^20, entry_size 16 and 256:
  - host-path (synchronous, wall clock) and device-path (CUDA events, enqueued back to back) updates of
    1, 1,024 and 65,536 random rows;
  - b200dpf_destroy + b200dpf_create of the same table (wall clock), the only way to change a row before;
  - the AES evaluation step at B = 512 with a 1,024-row device update between every two steps, against
    the same steps with no updates (CUDA events over the whole loop).
The card name and power limit are read in the same run.  Writes one JSON object to stdout and, with
--out DIR, to DIR/update_rows.json.

    python tools/gpu_update_rows.py --out results/
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
sys.path.insert(0, os.path.join(ROOT, "gpu-dpf_b200"))
import b200dpf  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def wall_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def event_ms(fn, reps, stream):
    """Mean time per call of `reps` calls enqueued back to back on `stream`."""
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(stream)
    for _ in range(reps):
        fn()
    t1.record(stream)
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def measure(n, e, steps):
    rng = np.random.RandomState(e)
    table = rng.randint(-2**31, 2**31, size=(n, e), dtype=np.int64).astype(np.int32)
    res = {"n": n, "entry_size": e, "host_ms": {}, "device_ms": {}}
    ctx = b200dpf.Context(table)
    stream = torch.cuda.Stream()
    for count in (1, 1024, 65536):
        idx = rng.randint(0, n, size=count).astype(np.int64)
        rows = rng.randint(-2**31, 2**31, size=(count, e), dtype=np.int64).astype(np.int32)
        ctx.update_rows(idx, rows)                       # grows the scratch
        res["host_ms"][count] = wall_ms(lambda: ctx.update_rows(idx, rows), 9)
        idx_d, rows_d = torch.from_numpy(idx).cuda(), torch.from_numpy(rows).cuda()
        torch.cuda.synchronize()
        res["device_ms"][count] = event_ms(
            lambda: ctx.update_rows_device(idx_d.data_ptr(), rows_d.data_ptr(), count, stream.cuda_stream), 50, stream)
    ctx.close()
    res["recreate_ms"] = wall_ms(lambda: b200dpf.Context(table).close(), 3)

    if e == 16:
        prf, batch = b200dpf.PRF_AES128, 512
        ctx = b200dpf.Context(table)
        alphas = rng.randint(0, n, size=batch)
        ka, _ = b200dpf.gen_batch(alphas, n, np.arange(batch) + 1, prf)
        keys = torch.from_numpy(ka).cuda()
        out = torch.empty((batch, e), dtype=torch.int32, device="cuda")
        idx_d = torch.from_numpy(rng.randint(0, n, size=1024).astype(np.int64)).cuda()
        rows_d = torch.from_numpy(rng.randint(-2**31, 2**31, size=(1024, e), dtype=np.int64).astype(np.int32)).cuda()
        torch.cuda.synchronize()
        s = stream.cuda_stream

        def step():
            ctx.eval_device(keys.data_ptr(), batch, prf, out.data_ptr(), s)

        def two_steps_with_update():
            step()
            ctx.update_rows_device(idx_d.data_ptr(), rows_d.data_ptr(), 1024, s)
            step()
        for _ in range(3):
            step()
        plain, mixed = [], []
        for _ in range(3):                               # alternate the two loops
            plain.append(event_ms(step, steps, stream))
            mixed.append(event_ms(two_steps_with_update, steps // 2, stream) / 2)
        res["aes_b512_step_ms"] = statistics.median(plain)
        res["aes_b512_step_with_update_every_2_ms"] = statistics.median(mixed)
        ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    report = {"card": card(), "results": [measure(1 << 20, e, args.steps) for e in (16, 256)]}
    line = json.dumps(report)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "update_rows.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
