"""Key generation on the host against tests/keygen_ref.py, a plain-Python restatement of the construction.

First the restatement's anchors: its ChaCha20 block function reproduces RFC 8439's test vectors, its mt19937
stream is std::mt19937's, and the construction driven by that stream reproduces the reference's own keys
(tests/golden/ref_checks_v1.npz) and the oracle's at every depth.  Driven by the ChaCha20 DRBG it reproduces
the stored early-terminated and XOR-shared keys, so those fixtures are checked rather than only recorded.

Then the engine against it, byte for byte, both servers, every PRF: gen_secure / gen_et / gen_xor and their
batched forms (one thread and every thread) at every depth of the kind, key_pack of those keys, the Python
layers with seeds longer than 44 bytes, a flip of every seed byte, and seeds chosen so the DRBG rejects even
draws (twice in a row, and at the last payload) and runs past 16 keystream blocks.  No GPU needed."""
import importlib.util
import os
import random
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402
import keygen_ref as R  # noqa: E402

PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)

# per kind: gen, gen_batch, key_pack of the engine
ENGINE = {
    "standard": (B.gen_secure, B.gen_batch_secure, B.key_pack),
    "et": (B.gen_et, B.gen_batch_et, B.key_pack_et),
    "xor": (B.gen_xor, B.gen_batch_xor, B.key_pack_xor),
}


def golden(name):
    return np.load(os.path.join(HERE, "golden", name))


def check_engine(kind, alphas, n, seeds, prf):
    """every host entry point of `kind` for these rows and seeds against the restatement"""
    gen, gen_batch, pack = ENGINE[kind]
    want = [R.gen(kind, a, n, s, prf) for a, s in zip(alphas, seeds)]
    for a, s, w in zip(alphas, seeds, want):
        ka, kb = gen(a, n, s, prf)
        assert np.array_equal(ka, w.a) and np.array_equal(kb, w.b), (kind, prf, n, a)
        assert pack(ka) == w.packed_a and pack(kb) == w.packed_b, (kind, prf, n, a)
    for nthreads in (1, 0):
        ka, kb = gen_batch(alphas, n, b"".join(bytes(s[:44]) for s in seeds), prf, nthreads=nthreads)
        for i, w in enumerate(want):
            assert np.array_equal(ka[i], w.a) and np.array_equal(kb[i], w.b), (kind, prf, n, alphas[i], nthreads)
    return want


# ---- anchors of the restatement ------------------------------------------------------------------------------

def test_chacha20_block_rfc8439_section_2_3_2():
    key = bytes(range(32))
    nonce = bytes.fromhex("000000090000004a00000000")
    assert R.chacha20_block_bytes(key, 1, nonce).hex() == (
        "10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e"
        "d2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e")


def test_chacha20_block_rfc8439_appendix_a1_vector_1():
    assert R.chacha20_block_bytes(bytes(32), 0, bytes(12)).hex() == (
        "76b8e0ada0f13d90405d6ae55386bd28bdd219b8a08ded1aa836efcc8b770dc7"
        "da41597c5157488d7724e03fb8d84a376a43b8f41518a11cc387b669b2ee6586")


def test_drbg_draws_are_the_keystream_in_order():
    """draw j is keystream bytes 16j .. 16j + 15 read as one little-endian integer: block 0 first, key seed[0:32],
    nonce seed[32:44], later seed bytes ignored"""
    seed = bytes((13 * i + 5) & 0xFF for i in range(60))
    stream = b"".join(R.chacha20_block_bytes(seed[:32], c, seed[32:44]) for c in range(3))
    g = R.ChaCha20Drbg(seed)
    for j in range(12):
        assert g.draw128() == int.from_bytes(stream[16 * j:16 * j + 16], "little"), j
    assert g.blocks == 3
    with pytest.raises(ValueError):
        R.ChaCha20Drbg(seed[:43])


def test_mt19937_stream_is_std_mt19937():
    """the 10000th output of a default-constructed std::mt19937 (seed 5489) is 4123659995 (C++11 26.5.5)"""
    g = R.MT19937Draws(5489)
    for _ in range(9999):
        g.output()
    assert g.output() == 4123659995


def test_mt_construction_reproduces_the_reference_keys():
    """the 48 key pairs the reference's CPU core generated (ref_checks_v1.npz, as SHA-256 of their bytes)"""
    spec = importlib.util.spec_from_file_location("make_golden_ref_checks",
                                                  os.path.join(HERE, "golden", "make_golden_ref_checks.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    checks = golden("ref_checks_v1.npz")
    cases = mk.gen_eval_inputs()
    assert len(cases) == 48 == len(checks["gen_keys_a_sha256"])
    for ci, (prf, n, alpha, seed32) in enumerate(cases):
        k = R.gen_mt(alpha, n, seed32, prf)
        assert np.array_equal(mk.sha256(k.a), checks["gen_keys_a_sha256"][ci]), ci
        assert np.array_equal(mk.sha256(k.b), checks["gen_keys_b_sha256"][ci]), ci


@pytest.mark.parametrize("prf", PRFS)
def test_mt_construction_matches_oracle_and_engine_every_depth(prf, oracle):
    """b200dpf_gen, b200dpf_gen_batch and the oracle's keygen (all the reference's generator) at depths 1 .. 32"""
    rng = random.Random(400 + prf)
    for depth in range(1, 33):
        n = 1 << depth
        alphas = R.edge_rows("standard", n, rng)
        seeds = [rng.getrandbits(32) for _ in alphas]
        want = [R.gen_mt(a, n, s, prf) for a, s in zip(alphas, seeds)]
        ba, bb = B.gen_batch(alphas, n, seeds, prf, nthreads=2)
        for i, (a, s, w) in enumerate(zip(alphas, seeds, want)):
            for ka, kb in (oracle.gen(a, n, s, prf), B.gen(a, n, s, prf), (ba[i], bb[i])):
                assert np.array_equal(ka, w.a) and np.array_equal(kb, w.b), (depth, a)


@pytest.mark.parametrize("kind,fixture", [("et", "et_v1.npz"), ("xor", "xor_v1.npz")])
def test_drbg_construction_reproduces_the_stored_keys(kind, fixture):
    data = golden(fixture)
    tags = sorted(k[:-len("_alpha")] for k in data.files if k.endswith("_alpha"))
    assert len(tags) == 8
    for tag in tags:
        prf = int(tag.split("_")[0][1:])
        n = 1 << int(tag.split("_n")[1])
        k = R.gen(kind, int(data[tag + "_alpha"]), n, data[tag + "_seed"].tobytes(), prf)
        assert np.array_equal(k.a, data[tag + "_key_a"]) and np.array_equal(k.b, data[tag + "_key_b"]), tag


# ---- the engine against the restatement ----------------------------------------------------------------------

@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("kind", list(R.KINDS))
def test_engine_keygen_every_depth(kind, prf):
    """gen / gen_batch (one thread, every thread) / key_pack of the kind at every depth it takes, n = 2^32
    included for standard keys, at row 0, n - 1, the lane edges and a random row"""
    rng = random.Random("%s %d" % (kind, prf))
    for depth in range(1, R.max_depth(kind) + 1):
        n = 1 << (depth + R.KINDS[kind].lane_bits)
        alphas = R.edge_rows(kind, n, rng)
        check_engine(kind, alphas, n, [rng.randbytes(44) for _ in alphas], prf)


@pytest.mark.parametrize("kind", list(R.KINDS))
def test_coverage_seeds_reach_the_drbg_edges(kind):
    """the seeds of keygen_ref.coverage_seeds do what they claim, and the engine follows the restatement through
    them for every PRF"""
    rng = random.Random(77)
    for cov in R.coverage_seeds(kind):
        n = 1 << (cov.depth + R.KINDS[kind].lane_bits)
        for prf in PRFS:
            alphas = R.edge_rows(kind, n, rng)
            for w in check_engine(kind, alphas, n, [cov.seed] * len(alphas), prf):
                rej, blocks = w.draws.odd_rejections, w.draws.blocks
                assert len(rej) == cov.depth - 1
                if cov.name == "depth 1":
                    assert rej == [] and blocks == 1          # 4 draws: two roots, two correction words
                elif cov.name == "two rejections":
                    assert rej[-1] >= 2
                else:
                    assert rej[-1] >= 1 and max(rej[:-1]) >= 2 and blocks > 16


@pytest.mark.parametrize("kind", list(R.KINDS))
def test_every_seed_byte_reaches_both_keys(kind):
    """flipping any one of the 44 seed bytes gives the keys the restatement predicts, and changes both"""
    gen = ENGINE[kind][0]
    n = 1 << (6 + R.KINDS[kind].lane_bits)
    alpha, prf = n // 2 + 5, PRFS[len(kind) % 4]
    seed = bytes((29 * i + 3) & 0xFF for i in range(44))
    base = R.gen(kind, alpha, n, seed, prf)
    for i in range(44):
        s = bytearray(seed)
        s[i] ^= 1 << (i % 8)
        want = R.gen(kind, alpha, n, bytes(s), prf)
        ka, kb = gen(alpha, n, bytes(s), prf)
        assert np.array_equal(ka, want.a) and np.array_equal(kb, want.b), i
        assert not np.array_equal(want.a, base.a) and not np.array_equal(want.b, base.b), i


def test_python_layers_use_the_first_44_seed_bytes():
    """dpf.DPF(...).gen(..., secure=True) of every kind and BinnedDPF.gen_in_bin: the restatement's keys for the
    first 44 bytes of a longer seed, whatever follows them"""
    import dpf
    seed = bytes((7 * i + 1) & 0xFF for i in range(64))
    other = seed[:44] + bytes(255 - b for b in seed[44:])
    for prf in PRFS:
        for kind, kw, n, alpha in (("standard", {}, 1 << 10, 1000), ("et", {"early_termination": True}, 1 << 10, 515),
                                   ("xor", {"xor": True}, 1 << 12, 4095)):
            want = R.gen(kind, alpha, n, seed[:44], prf)
            d = dpf.DPF(prf=prf, **kw)
            for s in (seed, other):
                k1, k2 = d.gen(alpha, n, seed=s, secure=True)
                assert np.array_equal(k1.numpy(), want.a) and np.array_equal(k2.numpy(), want.b), (kind, prf)
        b = dpf.BinnedDPF(prf=prf)
        b.bin_sizes = [2, 1 << 9, 1 << 20]         # what eval_init records; gen_in_bin needs no device
        for g, n in enumerate(b.bin_sizes):
            want = R.gen("standard", n - 1 - g, n, seed[:44], prf)
            k1, k2 = b.gen_in_bin(g, n - 1 - g, seed=seed, secure=True)
            assert np.array_equal(k1.numpy(), want.a) and np.array_equal(k2.numpy(), want.b), (g, prf)
