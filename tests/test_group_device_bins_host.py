"""Grouped evaluation from a device-resident bin list (b200dpf_group_eval_device_bins) on the host: the symbols, the
argument checks that need no device, and the Python layers, which refuse wrong shapes, dtypes and host-resident bins
before the library is called.  No GPU needed."""
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

ECUDA, ESTATE = -2, -4


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_symbols_present():
    L = C.CDLL(B.LIB_PATH)
    for name in ("b200dpf_group_eval_device_bins", "b200dpf_group_plan_lists"):
        assert name in B.SYMBOLS
        assert hasattr(L, name)


def test_not_a_grouped_context_is_estate():
    L = B.lib()
    assert L.b200dpf_group_eval_device_bins(None, C.c_void_p(16), C.c_void_p(16), 1, B.PRF_AES128, C.c_void_p(16), None,
                                            None) == ESTATE
    assert "not a grouped context" in L.b200dpf_last_error().decode()
    counts = np.zeros(4, np.int64)
    assert L.b200dpf_group_plan_lists(None, 0, counts, C.c_void_p(16), 0, C.c_void_p(16), 0, C.c_void_p(16), 0) == ESTATE


def test_refusals_match_the_host_bin_path():
    """a null context is refused before any buffer or count is looked at, as b200dpf_group_eval_device does"""
    L = B.lib()
    bins = np.zeros(1, np.int32)
    for nkeys in (0, 1, 1 << 25):
        assert L.b200dpf_group_eval_device_bins(None, None, None, nkeys, 9, None, None, None) == ESTATE
        msg_bins = L.b200dpf_last_error().decode()
        assert L.b200dpf_group_eval_device(None, None, bins, nkeys, 9, None, None) == ESTATE
        assert L.b200dpf_last_error().decode() == msg_bins


def test_group_context_names_itself():
    ctx = B.GroupContext.__new__(B.GroupContext)    # no device: a context that was never created
    ctx.handle = C.c_void_p()
    with pytest.raises(B.B200DPFError, match=r"b200dpf_group_eval_device_bins failed \(-4\).*not a grouped context"):
        ctx.eval_device_bins(16, 16, 1, B.PRF_AES128, 16)
    with pytest.raises(B.B200DPFError, match=r"b200dpf_group_plan_lists failed \(-4\)"):
        ctx.plan_lists(True)


@pytest.mark.skipif(_has_gpu(), reason="checks the behaviour without a CUDA device")
def test_fails_cleanly_without_device():
    """without a device no grouped context can be made (ECUDA, as for every GPU entry point), and the entry point
    refuses the missing context"""
    L = B.lib()
    h = C.c_void_p()
    table = np.zeros((8, 4), np.int32)
    ptrs = (C.c_void_p * 1)(table.ctypes.data)
    assert L.b200dpf_group_create(C.byref(h), ptrs, np.array([8], np.int64), 1, 4, 0) == ECUDA
    assert "no CUDA device" in L.b200dpf_last_error().decode()
    assert not h.value
    assert L.b200dpf_group_eval_device_bins(h, C.c_void_p(16), C.c_void_p(16), 1, B.PRF_AES128, C.c_void_p(16), None,
                                            None) == ESTATE


def test_dpf_cpp_refuses_an_empty_buffer_list():
    pytest.importorskip("torch")
    import dpf
    with pytest.raises(RuntimeError, match="empty buffer list"):
        dpf.dpf_cpp.group_eval_device_bins(16, 16, 1, [], B.PRF_AES128, 16, 0, 0)


def test_binned_dpf_refuses_before_the_library():
    """the refusals come first: a call that got past them would fail in dpf_cpp on the empty buffer list"""
    torch = pytest.importorskip("torch")
    import dpf
    d = dpf.BinnedDPF(prf=dpf.DPF.PRF_AES128)
    d.buffers = []
    d.table_effective_entry_size = 16
    keys = torch.zeros((3, 524), dtype=torch.int32)
    for bad in (keys, keys[:, :500], keys.long(), keys[0]):                    # host keys, wrong shape or dtype
        with pytest.raises(Exception, match=r"BinnedDPF\.eval_gpu_device_bins: keys_dev must be a contiguous int32 \[B, 524\]"):
            d.eval_gpu_device_bins(bad, torch.zeros(3, dtype=torch.int32))
