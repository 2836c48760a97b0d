"""GPU key generation against tests/keygen_ref.py, the plain-Python restatement that test_keygen_ref_host.py
anchors to RFC 8439 and the reference's keys: b200dpf_gen_batch_gpu (_et, _xor) at every depth of each kind,
n = 2^32 included, into host and device memory, and b200dpf_group_gen_queries_device in both formats, for every
PRF and both servers, byte for byte.  The seeds include keygen_ref.coverage_seeds, so the device's DRBG rejects
even draws, twice in a row and at the last payload, and runs past 16 keystream blocks."""
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

pytestmark = pytest.mark.gpu
PRFS = (B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128)
GPU_GEN = {"standard": B.gen_batch_gpu, "et": B.gen_batch_gpu_et, "xor": B.gen_batch_gpu_xor}
SENTINEL = 0xA5

# bins of a grouped context per kind: two depth-1 bins, a depth-2 bin (for the coverage seeds), one deep bin and
# one in between; one column per row keeps the deep bin's table small
BINS = {
    "standard": [2, 4, 1 << 20, 64, 2],
    "et": [8, 16, 1 << 22, 256, 8],
    "xor": [256, 512, 1 << 20, 1 << 10, 256],
}
GROUP_KW = {"standard": {}, "et": {"early_termination": True}, "xor": {"xor": True}}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("kind", list(R.KINDS))
def test_gen_batch_gpu_every_depth(torch_cuda, kind, prf):
    """every depth of the kind at row 0, n - 1, the lane edges and a random row, plus the coverage seeds at their
    depths; host outputs and device outputs (filled with -1 first, so every word must be written)"""
    torch = torch_cuda
    rng = random.Random("gpu %s %d" % (kind, prf))
    coverage = {c.depth: c.seed for c in R.coverage_seeds(kind)}
    for depth in range(1, R.max_depth(kind) + 1):
        n = 1 << (depth + R.KINDS[kind].lane_bits)
        alphas = R.edge_rows(kind, n, rng)
        seeds = [rng.randbytes(44) for _ in alphas]
        if depth in coverage:
            alphas, seeds = alphas * 2, seeds + [coverage[depth]] * len(alphas)
        want = [R.gen(kind, a, n, s, prf) for a, s in zip(alphas, seeds)]
        want_a, want_b = np.stack([w.a for w in want]), np.stack([w.b for w in want])
        ga, gb = GPU_GEN[kind](alphas, n, b"".join(seeds), prf)
        assert np.array_equal(ga, want_a) and np.array_equal(gb, want_b), depth
        da = torch.full((len(alphas), B.KEY_WORDS), -1, dtype=torch.int32, device="cuda")
        db = torch.full_like(da, -1)
        GPU_GEN[kind](alphas, n, b"".join(seeds), prf, out_ptrs=(da.data_ptr(), db.data_ptr()))
        torch.cuda.synchronize()
        assert np.array_equal(da.cpu().numpy(), want_a) and np.array_equal(db.cpu().numpy(), want_b), depth


@pytest.fixture(scope="module")
def contexts(torch_cuda):
    ctxs = {kind: B.GroupContext([np.zeros((n, 1), np.int32) for n in sizes], **GROUP_KW[kind])
            for kind, sizes in BINS.items()}
    yield ctxs
    for ctx in ctxs.values():
        ctx.close()


def query_inputs(kind, nq, rng):
    """alphas int64 [nq, nbins] -- query 0 all rows 0, query 1 all -1 (row n - 1 of every bin), the rest any int64 --
    and seeds uint8 [nq, nbins, 44], with the coverage seed of a bin's depth in the first and the last query"""
    nbins = len(BINS[kind])
    alphas = np.array([[rng.randrange(-2**63, 2**63) for _ in range(nbins)] for _ in range(nq)], np.int64)
    alphas[0] = 0
    if nq > 1:
        alphas[1] = -1
    seeds = np.frombuffer(rng.randbytes(nq * nbins * 44), np.uint8).reshape(nq, nbins, 44).copy()
    coverage = {c.depth: c.seed for c in R.coverage_seeds(kind)}
    for g, n in enumerate(BINS[kind]):
        seed = coverage.get(R.depth_of(kind, n))
        if seed is not None:
            seeds[0, g] = seeds[nq - 1, g] = np.frombuffer(seed, np.uint8)
    return alphas, seeds


def gen_device(torch, ctx, alphas, seeds, prf, compact, sentinel=64):
    """both servers' query batches from GroupContext.gen_queries_device as host bytes, into buffers filled with
    SENTINEL whose `sentinel` bytes after the last query must stay untouched"""
    nq, nbins = alphas.shape
    size = nq * (ctx.query_bytes if compact else nbins * B.KEY_WORDS * 4)
    outs = [torch.full((size + sentinel,), SENTINEL, dtype=torch.uint8, device="cuda") for _ in range(2)]
    a_dev = torch.from_numpy(alphas).cuda()
    s_dev = torch.from_numpy(seeds).cuda()
    st = torch.cuda.current_stream()
    ctx.gen_queries_device(a_dev.data_ptr(), s_dev.data_ptr(), nq, prf, outs[0].data_ptr(), outs[1].data_ptr(),
                           st.cuda_stream, compact=compact)
    st.synchronize()
    res = []
    for o in outs:
        h = o.cpu().numpy()
        assert (h[size:] == SENTINEL).all(), "bytes after the last query written"
        res.append(h[:size])
    return res


@pytest.mark.parametrize("nq", [1, 33])
@pytest.mark.parametrize("prf", PRFS)
@pytest.mark.parametrize("kind", list(R.KINDS))
def test_gen_queries_device_every_key(torch_cuda, contexts, kind, prf, nq):
    """key (q, g) of both servers' batches, wire and compact, is the restatement's key for row alphas[q, g] mod n_g
    of bin g from seeds[q, g]"""
    ctx = contexts[kind]
    sizes = BINS[kind]
    alphas, seeds = query_inputs(kind, nq, random.Random("queries %s %d %d" % (kind, prf, nq)))
    want = [[R.gen(kind, int(alphas[q, g]) % n, n, seeds[q, g].tobytes(), prf) for g, n in enumerate(sizes)]
            for q in range(nq)]
    wire_a, wire_b = gen_device(torch_cuda, ctx, alphas, seeds, prf, compact=False)
    for out, srv in ((wire_a, "a"), (wire_b, "b")):
        got = out.view(np.int32).reshape(nq, len(sizes), B.KEY_WORDS)
        for q in range(nq):
            for g in range(len(sizes)):
                assert np.array_equal(got[q, g], getattr(want[q][g], srv)), (srv, q, g)
    compact_a, compact_b = gen_device(torch_cuda, ctx, alphas, seeds, prf, compact=True)
    for out, srv in ((compact_a, "packed_a"), (compact_b, "packed_b")):
        got = out.reshape(nq, ctx.query_bytes)
        for q in range(nq):
            assert got[q].tobytes() == b"".join(getattr(w, srv) for w in want[q]), (srv, q)
