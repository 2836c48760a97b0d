"""Generate tests/golden/ref_checks_v1.npz: what the original project's CPU core returns for the
inputs of the oracle-vs-reference tests in tests/test_oracle.py, so those comparisons run
anywhere, without the original sources.

Run where the original project is available, after `make -C oracle ref` built oracle/_ref/libdpfref.so:

    python tests/golden/make_golden_ref_checks.py

Keys, share vectors and the PRF outputs of each PRF are stored as SHA-256 digests of their
little-endian bytes (an exact comparison at 32 bytes per array); everything else is stored as is.
"""
import hashlib
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle as O  # noqa: E402
from common import formula_table  # noqa: E402

PATH = os.path.join(ROOT, "tests", "golden", "ref_checks_v1.npz")


def sha256(v):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(v, "<i4").tobytes()).digest(), np.uint8)


def prf_inputs():
    """Seeds of test_oracle_matches_reference_prf, in order."""
    r = random.Random(7)
    return [r.getrandbits(128) for _ in range(200)]


def gen_eval_inputs():
    """(prf, n, alpha, seed32) of test_oracle_matches_reference_gen_and_eval, in order."""
    r = random.Random(11)
    cases = []
    for prf in range(4):
        for n in (2, 4, 256, 2048):
            for _ in range(3):
                alpha, seed32 = r.randrange(n), r.getrandbits(32)
                cases.append((prf, n, alpha, seed32))
    return cases


def main():
    ref = O.Ref()
    out = {}
    seeds = prf_inputs()
    prf_out = np.zeros((len(seeds), 4, 2, 2), np.uint64)          # [seed][prf][pos][lo, hi]
    for si, s in enumerate(seeds):
        for prf in range(4):
            for pos in (0, 1):
                v = ref.prf(prf, s, pos)
                prf_out[si, prf, pos] = (v & (2**64 - 1), v >> 64)
    out["prf_out_sha256"] = np.stack([sha256(prf_out[:, prf].view(np.int32)) for prf in range(4)])

    cases = gen_eval_inputs()
    keys_a = np.zeros((len(cases), 32), np.uint8)
    keys_b = np.zeros((len(cases), 32), np.uint8)
    full_a = np.zeros((len(cases), 32), np.uint8)
    flat_b = np.zeros((len(cases), 3, 2), np.uint64)              # at indices 0, alpha, n - 1
    for ci, (prf, n, alpha, seed32) in enumerate(cases):
        ka, kb = ref.gen(alpha, n, seed32, prf)
        keys_a[ci], keys_b[ci] = sha256(ka), sha256(kb)
        full_a[ci] = sha256(ref.eval_full(ka, prf))
        for j, idx in enumerate((0, alpha, n - 1)):
            v = ref.eval_flat(kb, idx, prf)
            flat_b[ci, j] = (v & (2**64 - 1), v >> 64)
    out.update(gen_keys_a_sha256=keys_a, gen_keys_b_sha256=keys_b, gen_full_a_sha256=full_a, gen_flat_b=flat_b)

    # the harness behind bench.py --impl reference: ref_eval_dot_mt over 3 threads
    n = 512
    t = formula_table(n, 16)
    keys = np.stack([ref.gen(i * 37 % n, n, 50 + i, 2)[0] for i in range(5)])
    out["harness_keys_sha256"] = sha256(keys)
    out["harness_dot"] = ref.eval_dot_mt(keys, 2, t, 0, n, 3)
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH), "bytes")


if __name__ == "__main__":
    main()
