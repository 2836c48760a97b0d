"""GPU kernel against GPU kernel: this engine vs the original project's own dpf_hybrid_kernel.
Same keys, same table, results must be bit-identical.  The original kernel's results were
recorded on an H100 by tests/golden/make_golden_refgpu.py into tests/golden/refgpu_v1.npz as
SHA-256 digests; the inputs are regenerated here from their seeds and checked against stored
digests too."""
import hashlib
import os

import numpy as np
import pytest

import b200dpf
from common import random_table, seeded_keys

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def refgpu():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refgpu_v1.npz"))


def _sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a, "<i4").tobytes()).digest()


@pytest.mark.parametrize("prf", [0, 1, 2, 3])
def test_same_results_as_reference_kernel(refgpu, prf):
    n, batch = 4096, 70
    table = random_table(n, 16, seed=prf, full_range=True)
    ka, kb, idx = seeded_keys(b200dpf.gen, n, batch, prf, seed=40 + prf)
    assert _sha256(np.concatenate([ka, kb])) == refgpu["keys_sha256_%d" % prf].tobytes(), "inputs changed"
    ctx = b200dpf.Context(table)
    got_a, got_b = ctx.eval(ka, prf), ctx.eval(kb, prf)
    ctx.close()
    assert _sha256(got_a) == refgpu["want_a_sha256_%d" % prf].tobytes()
    assert _sha256(got_b) == refgpu["want_b_sha256_%d" % prf].tobytes()
    assert np.array_equal((got_a.astype(np.uint32) - got_b.astype(np.uint32)).astype(np.int32), table[idx])


def test_entry_size_and_short_batch_like_reference(refgpu):
    n, batch, entry, prf = 1024, 5, 7, 3
    table = random_table(n, entry, seed=9)
    ka, _, _ = seeded_keys(b200dpf.gen, n, batch, prf, seed=9)
    assert _sha256(ka) == refgpu["short_keys_sha256"].tobytes(), "inputs changed"
    ctx = b200dpf.Context(table)
    assert _sha256(ctx.eval(ka, prf)) == refgpu["short_want_sha256"].tobytes()
    ctx.close()
