"""Writes tests/golden/et_v1.npz: early-terminated keys from fixed seeds and their share vectors.

    python tests/golden/make_golden_et.py

For every PRF and n in {2^10, 2^14}: one key pair (alpha and the 44-byte seed are stored too) and
both servers' shares of every row, computed by the per-index oracle (tests/et_oracle.py).  The file
pins the key format and the construction; tests/test_et_host.py checks the engine against it.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle"), os.path.dirname(HERE)]

import b200dpf  # noqa: E402
import et_oracle  # noqa: E402
import oracle  # noqa: E402


def main():
    orc = oracle.Oracle()
    data = {}
    for prf in range(4):
        for logn in (10, 14):
            n = 1 << logn
            alpha = (0x9E3779B1 * (prf + 1) * logn) % n
            seed = bytes((7 * i + 13 * prf + logn) & 0xFF for i in range(44))
            a, b = b200dpf.gen_et(alpha, n, seed, prf)
            tag = "p%d_n%d" % (prf, logn)
            data[tag + "_alpha"] = np.int64(alpha)
            data[tag + "_seed"] = np.frombuffer(seed, np.uint8)
            data[tag + "_key_a"] = a
            data[tag + "_key_b"] = b
            data[tag + "_share_a"] = et_oracle.eval_full_flat_et(orc, a, prf)
            data[tag + "_share_b"] = et_oracle.eval_full_flat_et(orc, b, prf)
    np.savez_compressed(os.path.join(HERE, "et_v1.npz"), **data)


if __name__ == "__main__":
    main()
