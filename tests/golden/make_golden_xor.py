"""Writes tests/golden/xor_v1.npz: XOR-shared keys from fixed seeds and their share bits.

    python tests/golden/make_golden_xor.py

For every PRF and n in {2^10, 2^14}: one key pair (alpha and the 44-byte seed are stored too) and
both servers' share bits of every row, packed 32 to a uint32 word, computed by the per-index oracle
(tests/xor_oracle.py).  The file pins the key format and the construction; tests/test_xor_host.py
checks the engine against it.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle"), os.path.dirname(HERE)]

import b200dpf  # noqa: E402
import oracle  # noqa: E402
import xor_oracle  # noqa: E402


def main():
    orc = oracle.Oracle()
    data = {}
    for prf in range(4):
        for logn in (10, 14):
            n = 1 << logn
            alpha = (0x9E3779B1 * (prf + 1) * logn) % n
            seed = bytes((11 * i + 17 * prf + logn) & 0xFF for i in range(44))
            a, b = b200dpf.gen_xor(alpha, n, seed, prf)
            tag = "p%d_n%d" % (prf, logn)
            data[tag + "_alpha"] = np.int64(alpha)
            data[tag + "_seed"] = np.frombuffer(seed, np.uint8)
            data[tag + "_key_a"] = a
            data[tag + "_key_b"] = b
            data[tag + "_bits_a"] = xor_oracle.pack_bits(xor_oracle.share_bits(orc, a, prf))
            data[tag + "_bits_b"] = xor_oracle.pack_bits(xor_oracle.share_bits(orc, b, prf))
    np.savez_compressed(os.path.join(HERE, "xor_v1.npz"), **data)


if __name__ == "__main__":
    main()
