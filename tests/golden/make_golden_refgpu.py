"""Generate tests/golden/refgpu_v1.npz: what the original project's own GPU kernel
(dpf_hybrid_kernel, built unmodified into oracle/_ref/ref_dpf_cpp.so by oracle/build_refgpu.py)
returns for the inputs of tests/test_gpu_vs_reference_gpu.py, so that comparison runs without
the original sources.

Run on a GPU machine where oracle/_ref/ref_dpf_cpp.so was built:

    python tests/golden/make_golden_refgpu.py [output.npz]

Tables and keys are regenerated from their seeds by the test.  Results and key batches are stored
as SHA-256 digests of their little-endian int32 bytes: an exact comparison, and a change of inputs
is told apart from a change of results.
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for sub in ("gpu-dpf_b200", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, sub))
import b200dpf  # noqa: E402
import refgpu  # noqa: E402
from common import random_table, seeded_keys  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "refgpu_v1.npz")


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, "<i4").tobytes()).digest(), np.uint8)


def same_results_inputs(prf):
    n, batch = 4096, 70
    table = random_table(n, 16, seed=prf, full_range=True)
    ka, kb, idx = seeded_keys(b200dpf.gen, n, batch, prf, seed=40 + prf)
    return table, ka, kb, idx


def short_batch_inputs():
    n, batch, entry, prf = 1024, 5, 7, 3
    table = random_table(n, entry, seed=9)
    ka, _, _ = seeded_keys(b200dpf.gen, n, batch, prf, seed=9)
    return table, ka, prf


def run_ref(prf, table, keys):
    ref = refgpu.RefGpuDPF(prf)
    ref.eval_init(torch.from_numpy(table))
    out = ref.eval_gpu([torch.from_numpy(k) for k in keys]).numpy()
    ref.close()
    return out


def main():
    if not refgpu.available():
        raise SystemExit("oracle/_ref/ref_dpf_cpp.so not built")
    out = {}
    for prf in range(4):
        table, ka, kb, _ = same_results_inputs(prf)
        out["want_a_sha256_%d" % prf] = digest(run_ref(prf, table, ka))
        out["want_b_sha256_%d" % prf] = digest(run_ref(prf, table, kb))
        out["keys_sha256_%d" % prf] = digest(np.concatenate([ka, kb]))
    table, ka, prf = short_batch_inputs()
    out["short_want_sha256"] = digest(run_ref(prf, table, ka))
    out["short_keys_sha256"] = digest(ka)
    out["device"] = np.array(torch.cuda.get_device_name(0))
    path = sys.argv[1] if len(sys.argv) > 1 else PATH
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
