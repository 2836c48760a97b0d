"""Batch-PIR query batches (b200dpf_group_eval_queries_device, b200dpf_group_query_bytes) on the host: the
symbols, the refusals that need no device, pack_queries' layout against key_pack of each kind at mixed bin
depths, and the Python layers, which refuse wrong shapes, dtypes and host tensors before the library is
called.  No GPU needed."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402

ESTATE = -4

# per kind suffix: bin sizes of mixed depths (from the smallest the kind takes), key generator
KINDS = {
    "": ([2, 64, 1 << 10, 8], lambda al, n, rng: B.gen_batch(al, n, rng.randint(0, 2**31, size=len(al)), B.PRF_AES128)),
    "_et": ([8, 64, 1 << 10, 32], lambda al, n, rng: B.gen_batch_et(al, n, rng.bytes(44 * len(al)), B.PRF_AES128)),
    "_xor": ([256, 1 << 12, 512, 1 << 10], lambda al, n, rng: B.gen_batch_xor(al, n, rng.bytes(44 * len(al)), B.PRF_AES128)),
}


def host_group_context(kind, sizes):
    """a GroupContext without a device: what pack_queries reads (its kind and bin sizes) and a null handle"""
    ctx = B.GroupContext.__new__(B.GroupContext)
    ctx.handle = C.c_void_p()
    ctx.kind = kind
    ctx.tables = [np.zeros((n, 1), np.int32) for n in sizes]
    return ctx


def test_symbols_present():
    L = C.CDLL(B.LIB_PATH)
    for name in ("b200dpf_group_query_bytes", "b200dpf_group_eval_queries_device"):
        assert name in B.SYMBOLS
        assert hasattr(L, name)
    assert (B.KEYS_WIRE, B.KEYS_COMPACT) == (0, 1)


def test_not_a_grouped_context():
    assert B.lib().b200dpf_group_query_bytes(None) == -1
    for fmt in (B.KEYS_WIRE, B.KEYS_COMPACT):
        assert B.lib().b200dpf_group_eval_queries_device(None, C.c_void_p(16), fmt, 1, B.PRF_AES128, C.c_void_p(16), None) == ESTATE
        assert "not a grouped context" in B.lib().b200dpf_last_error().decode()
    ctx = host_group_context("", [2])
    assert ctx.query_bytes == -1
    with pytest.raises(B.B200DPFError, match=r"b200dpf_group_eval_queries_device failed \(-4\).*not a grouped context"):
        ctx.eval_queries_device(16, 1, B.PRF_AES128, 16, compact=True)


@pytest.mark.parametrize("kind", list(KINDS))
def test_pack_queries_layout(kind):
    """query q is key_pack<kind>(keys[q, g]) for g = 0, 1, .. back to back, each at its bin's depth"""
    sizes, gen = KINDS[kind]
    rng = np.random.RandomState(len(kind))
    nq = 3
    keys = np.zeros((nq, len(sizes), B.KEY_WORDS), np.int32)
    for g, n in enumerate(sizes):
        keys[:, g] = gen(rng.randint(0, n, size=nq).astype(np.int64), n, rng)[0]
    ctx = host_group_context(kind, sizes)
    packed = ctx.pack_queries(keys)
    lane_bits = B.KINDS[kind][0]
    widths = [32 + 64 * (n.bit_length() - 1 - lane_bits) for n in sizes]
    assert packed.dtype == np.uint8 and packed.shape == (nq, sum(widths))
    assert all(w % 16 == 0 for w in widths)
    for q in range(nq):
        want = b"".join(B._key_pack(kind, keys[q, g]) for g in range(len(sizes)))
        assert packed[q].tobytes() == want
    assert [B.lib().b200dpf_key_packed_size(n.bit_length() - 1 - lane_bits) for n in sizes] == widths


def test_pack_queries_refusals():
    sizes, gen = KINDS["_xor"]
    rng = np.random.RandomState(5)
    ctx = host_group_context("_xor", sizes)
    keys = np.zeros((2, len(sizes), B.KEY_WORDS), np.int32)
    for g, n in enumerate(sizes):
        keys[:, g] = gen(np.zeros(2, np.int64), n, rng)[0]
    with pytest.raises(ValueError, match=r"pack_queries: keys must be int32 \[Q, 4, 524\]"):
        ctx.pack_queries(keys[:, :3])
    with pytest.raises(ValueError, match=r"pack_queries: keys must be"):
        ctx.pack_queries(keys[0])
    swapped = keys.copy()
    swapped[1, 0], swapped[1, 1] = keys[1, 1], keys[1, 0]          # keys for the wrong bins' sizes
    with pytest.raises(ValueError, match=r"key 0 of query 1 is for another bin size"):
        ctx.pack_queries(swapped)
    std = host_group_context("", sizes)                            # XOR-shared keys on a standard context
    with pytest.raises(B.B200DPFError, match=r"b200dpf_key_pack failed"):
        std.pack_queries(keys)


def test_dpf_cpp_surface():
    pytest.importorskip("torch")
    import dpf
    cpp = dpf.dpf_cpp
    assert hasattr(cpp, "group_eval_queries_device") and hasattr(cpp, "group_query_bytes")
    with pytest.raises(RuntimeError, match="empty buffer list"):
        cpp.group_query_bytes([])
    with pytest.raises(RuntimeError, match="empty buffer list"):
        cpp.group_eval_queries_device(16, 1, [], B.PRF_AES128, 16, 0, True)


def test_binned_dpf_refuses_before_the_library():
    """the refusals come first: a call that got past them would fail in dpf_cpp on the empty buffer list"""
    torch = pytest.importorskip("torch")
    import dpf
    d = dpf.BinnedDPF(prf=dpf.DPF.PRF_AES128)
    with pytest.raises(Exception, match=r"BinnedDPF\.eval_queries_device: must call `eval_init` first"):
        d.eval_queries_device(torch.zeros((1, 3, 524), dtype=torch.int32))
    d.buffers = []
    d.bin_sizes = [2, 64, 1 << 10]
    d.table_effective_entry_size = 16
    keys = torch.zeros((2, 3, 524), dtype=torch.int32)
    for bad in (keys, keys.long(), keys.float(), keys.to(torch.uint8), keys[:, :, :500], "keys"):   # host tensors, wrong dtypes
        with pytest.raises(Exception, match=r"BinnedDPF\.eval_queries_device: keys_dev must be a contiguous CUDA tensor "
                                            r"on cuda:0, int32 \[Q, 3, 524\] or uint8 \[Q, query_bytes\]"):
            d.eval_queries_device(bad)
