"""GPU key generation for every kind (b200dpf_gen_batch_gpu_et, _xor) and batch-PIR query generation
(b200dpf_group_gen_queries_device) on the host: the symbols, the refusals that need no device, in their order,
and the Python layers, which refuse wrong shapes, dtypes and host tensors before the library is called.  No GPU
needed."""
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

EINVAL, ECUDA, ESTATE = -1, -2, -4
NEW = ("b200dpf_gen_batch_gpu_et", "b200dpf_gen_batch_gpu_xor", "b200dpf_group_gen_queries_device")

# per kind suffix: (smallest n, largest n, CPU entry point the ECUDA message names)
RANGES = {
    "": (2, 1 << 32, "b200dpf_gen_batch_secure"),
    "_et": (8, 1 << 31, "b200dpf_gen_batch_et"),
    "_xor": (256, 1 << 31, "b200dpf_gen_batch_xor"),
}


def test_symbols_present():
    L = C.CDLL(B.LIB_PATH)
    for name in NEW:
        assert name in B.SYMBOLS
        assert hasattr(L, name)


def test_not_a_grouped_context():
    """ESTATE on a null context comes first, for every format and whatever else is wrong"""
    gen = B.lib().b200dpf_group_gen_queries_device
    for fmt in (B.KEYS_WIRE, B.KEYS_COMPACT, 7):
        assert gen(None, C.c_void_p(16), C.c_void_p(16), 1, B.PRF_AES128, fmt, C.c_void_p(16), C.c_void_p(16), None) == ESTATE
        assert "not a grouped context" in B.lib().b200dpf_last_error().decode()
        assert gen(None, None, None, 0, 9, fmt, None, C.c_void_p(3), None) == ESTATE
    ctx = B.GroupContext.__new__(B.GroupContext)
    ctx.handle = C.c_void_p()
    with pytest.raises(B.B200DPFError, match=r"b200dpf_group_gen_queries_device failed \(-4\).*not a grouped context"):
        ctx.gen_queries_device(16, 16, 1, B.PRF_AES128, 16, 16, compact=True)


@pytest.mark.parametrize("kind", list(RANGES))
def test_gen_batch_gpu_refusals(kind):
    """n and every alpha are checked, per kind, before a device is looked for; without a device the message
    names the CPU entry point of the same keys"""
    n_min, n_max, cpu = RANGES[kind]
    fn = getattr(B, "gen_batch_gpu" + kind)
    name = "b200dpf_gen_batch_gpu" + kind
    for n in (n_min // 2, n_max * 2, n_min * 3, 0, -n_min):
        with pytest.raises(B.B200DPFError, match=r"%s failed \(-1\): n=%d must be a power of two in \[%d, 2\^%d\]"
                           % (name, n, n_min, n_max.bit_length() - 1)):
            fn([0], n, bytes(44), B.PRF_AES128)
    for alpha in (-1, n_min, 1 << 40):
        with pytest.raises(B.B200DPFError, match=r"%s failed \(-1\): gen_batch_gpu%s: alpha\[1\]=%d out of range"
                           % (name, kind, alpha)):
            fn([0, alpha], n_min, bytes(88), B.PRF_AES128)
    with pytest.raises(B.B200DPFError, match=r"unknown prf id 4"):
        fn([0], n_min, bytes(44), 4)
    assert fn([], n_min, b"", B.PRF_AES128)[0].shape == (0, B.KEY_WORDS)   # nothing to do: no device needed
    L = B.lib()
    a = np.zeros(B.KEY_WORDS, np.int32)
    assert getattr(L, name)(np.zeros(1, np.int64), None, 1, n_min, B.PRF_AES128, 0, a.ctypes.data_as(C.c_void_p),
                            a.ctypes.data_as(C.c_void_p)) == EINVAL
    assert "bad gen_batch_gpu%s argument" % kind in L.b200dpf_last_error().decode()


@pytest.mark.parametrize("kind", list(RANGES))
def test_gen_batch_gpu_without_device(kind):
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("a CUDA device is present")
    except ImportError:
        pass
    n_min, _, cpu = RANGES[kind]
    with pytest.raises(B.B200DPFError, match=r"failed \(-2\): no CUDA device available \(use %s on the CPU\)" % cpu):
        getattr(B, "gen_batch_gpu" + kind)([0, n_min - 1], n_min, bytes(88), B.PRF_AES128)


def test_dpf_cpp_surface():
    pytest.importorskip("torch")
    import dpf
    cpp = dpf.dpf_cpp
    assert hasattr(cpp, "group_gen_queries_device")
    with pytest.raises(RuntimeError, match="empty buffer list"):
        cpp.group_gen_queries_device(16, 16, 1, [], B.PRF_AES128, 16, 16, 0, True)
    with pytest.raises(RuntimeError, match="empty buffer list"):
        cpp.group_gen_queries_device(16, 16, 1, [], B.PRF_AES128, 16, 16, 0)


def test_binned_dpf_refuses_before_the_library():
    """the refusals come first: a call that got past them would fail in dpf_cpp on the empty buffer list"""
    torch = pytest.importorskip("torch")
    import dpf
    d = dpf.BinnedDPF(prf=dpf.DPF.PRF_AES128)
    with pytest.raises(Exception, match=r"BinnedDPF\.gen_queries_device: must call `eval_init` first"):
        d.gen_queries_device(torch.zeros((1, 3), dtype=torch.int64))
    d.buffers = []
    d.bin_sizes = [2, 64, 1 << 10]
    d.table_effective_entry_size = 16
    idx = torch.zeros((2, 3), dtype=torch.int64)
    for bad in (idx, idx.int(), idx.float(), idx[:, :2], idx.reshape(6), idx.reshape(2, 3, 1), "idx"):
        with pytest.raises(Exception, match=r"BinnedDPF\.gen_queries_device: indices_dev must be a contiguous int64 "
                                            r"\[Q, 3\] tensor on cuda:0"):
            d.gen_queries_device(bad)
    # BinnedDPF keeps refusing the other kinds of key: they are reached through GroupContext / dpf_cpp
    for kw in ("early_termination", "xor"):
        with pytest.raises(Exception, match="BinnedDPF has no"):
            dpf.BinnedDPF(prf=dpf.DPF.PRF_AES128, **{kw: True})
