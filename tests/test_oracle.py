"""The CPU oracle against the golden vectors produced by the original project's CPU core.  No GPU."""
import hashlib
import os
import random

import numpy as np
import pytest

from common import dot_u32, formula_table


@pytest.fixture(scope="module")
def ref_checks():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_checks_v1.npz"))

# values printed by the unmodified reference for seed 0x0123456789abcdef_fedcba9876543210 (SURVEY.md section 8c)
SURVEY_SEED = 0x0123456789ABCDEFFEDCBA9876543210
SURVEY_KAT = {
    (0, 0): 0xDA740DA740DA72CD258BF258BF259DB2, (0, 1): 0xDB97530ECA8640BD2468ACF13579CFC3,
    (1, 0): 0x5FBDA2E3F234E6B2B441D17E91810713, (1, 1): 0x96BFF27E59D21AF7115FC04F9F69A796,
    (2, 0): 0x63B38CD27C19ADE41BA01054F62962A9, (2, 1): 0x4EF8FD229FC67648B29DE9F00E19B12A,
    (3, 0): 0x13F02B85CF6357E3A3716CB94327E294, (3, 1): 0x18B5654ACFC155AA5008DAAB2FCED214,
}


def test_aes_fips197_c1(oracle):
    key = bytes(range(16))
    pt = bytes.fromhex("00112233445566778899aabbccddeeff")
    assert oracle.aes128_encrypt(key, pt).hex() == "69c4e0d86a7b0430d8cdb78070b4c55a"


def test_prf_survey_values(oracle):
    for (prf, pos), want in SURVEY_KAT.items():
        assert oracle.prf(prf, SURVEY_SEED, pos) == want


def test_prf_golden(oracle, golden):
    seeds, outs = golden["kat_seed"], golden["kat_out"]
    for si in range(seeds.shape[0]):
        s = int(seeds[si, 0]) | (int(seeds[si, 1]) << 64)
        for prf in range(4):
            for pos in (0, 1):
                want = int(outs[prf, si, pos, 0]) | (int(outs[prf, si, pos, 1]) << 64)
                assert oracle.prf(prf, s, pos) == want


def test_gen_golden(oracle, golden):
    meta = golden["case_meta"]
    for ci, (prf, n, alpha, seed32) in enumerate(meta):
        ka, kb = oracle.gen(int(alpha), int(n), int(seed32), int(prf))
        assert np.array_equal(ka, golden["keys_a"][ci])
        assert np.array_equal(kb, golden["keys_b"][ci])


def test_eval_golden(oracle, golden):
    meta = golden["case_meta"]
    for ci, (prf, n, alpha, seed32) in enumerate(meta):
        prf, n = int(prf), int(n)
        ka, kb = golden["keys_a"][ci], golden["keys_b"][ci]
        sa = oracle.eval_full(ka, prf, tree=True)
        sb = oracle.eval_full(kb, prf, tree=True)
        if n <= 1024:
            assert np.array_equal(sa, golden["share_a_%d" % ci])
            assert np.array_equal(sb, golden["share_b_%d" % ci])
            assert np.array_equal(oracle.eval_full(ka, prf, tree=False), sa)
        t = formula_table(n, 16)
        assert np.array_equal(oracle.eval_dot(ka, prf, t)[0], golden["dots_a"][ci])
        assert np.array_equal(oracle.eval_dot(kb, prf, t)[0], golden["dots_b"][ci])
        assert np.array_equal(dot_u32(sa[None, :], t)[0], golden["dots_a"][ci])


def test_shard_partials_add_up(oracle, golden):
    """Entry-range shards (SURVEY.md section 8e): partial sums over disjoint
    breadth-first leaf ranges add to the whole inner product mod 2^32."""
    meta = golden["case_meta"]
    for ci, (prf, n, alpha, seed32) in enumerate(meta):
        n = int(n)
        if n != 1024:
            continue
        t = formula_table(n, 16)
        for shards in (2, 8):
            acc = np.zeros(16, np.uint32)
            for r in range(shards):
                acc += oracle.eval_dot_shard(golden["keys_a"][ci], int(prf), t, r * n // shards, n // shards).astype(np.uint32)
            assert np.array_equal(acc.astype(np.int32), golden["dots_a"][ci])


def test_dot_range_matches_full(oracle, golden):
    ci = [i for i, m in enumerate(golden["case_meta"]) if m[1] == 1024][0]
    prf = int(golden["case_meta"][ci][0])
    t = formula_table(1024, 16)
    a = oracle.eval_dot_range(golden["keys_a"][ci], prf, t, 0, 512).astype(np.uint32)
    b = oracle.eval_dot_range(golden["keys_a"][ci], prf, t, 512, 512).astype(np.uint32)
    assert np.array_equal((a + b).astype(np.int32)[0], golden["dots_a"][ci])


# ---- against the original project's CPU core (outputs stored by tests/golden/make_golden_ref_checks.py)

def _sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a, "<i4").tobytes()).digest()


def _u128(lohi):
    return int(lohi[0]) | (int(lohi[1]) << 64)


def test_oracle_matches_reference_prf(oracle, ref_checks):
    r = random.Random(7)
    seeds = [r.getrandbits(128) for _ in range(200)]
    for prf in range(4):
        got = np.zeros((len(seeds), 2, 2), np.uint64)          # [seed][pos][lo, hi]
        for si, s in enumerate(seeds):
            for pos in (0, 1):
                v = oracle.prf(prf, s, pos)
                got[si, pos] = (v & (2**64 - 1), v >> 64)
        assert hashlib.sha256(got.tobytes()).digest() == ref_checks["prf_out_sha256"][prf].tobytes(), prf


def test_oracle_matches_reference_gen_and_eval(oracle, ref_checks):
    r = random.Random(11)
    ci = 0
    for prf in range(4):
        for n in (2, 4, 256, 2048):
            for _ in range(3):
                alpha, seed32 = r.randrange(n), r.getrandbits(32)
                ka, kb = oracle.gen(alpha, n, seed32, prf)
                assert _sha256(ka) == ref_checks["gen_keys_a_sha256"][ci].tobytes(), (prf, n, alpha)
                assert _sha256(kb) == ref_checks["gen_keys_b_sha256"][ci].tobytes(), (prf, n, alpha)
                assert _sha256(oracle.eval_full(ka, prf)) == ref_checks["gen_full_a_sha256"][ci].tobytes(), (prf, n, alpha)
                for j, idx in enumerate((0, alpha, n - 1)):
                    assert oracle.eval_flat(kb, idx, prf) == _u128(ref_checks["gen_flat_b"][ci, j]), (prf, n, idx)
                ci += 1
    assert ci == ref_checks["gen_keys_a_sha256"].shape[0]


def test_reference_baseline_harness(oracle, ref_checks):
    """ref_eval_dot_mt (the --impl reference timing leg) computes the same inner product as the oracle."""
    n = 512
    t = formula_table(n, 16)
    keys = np.stack([oracle.gen(i * 37 % n, n, 50 + i, 2)[0] for i in range(5)])
    assert _sha256(keys) == ref_checks["harness_keys_sha256"].tobytes()
    assert np.array_equal(ref_checks["harness_dot"], oracle.eval_dot(keys, 2, t))
    import oracle as O
    if O.Ref.available():      # where the reference core was built, also run the code bench.py times
        assert np.array_equal(O.Ref().eval_dot_mt(keys, 2, t, 0, n, 3), ref_checks["harness_dot"])
