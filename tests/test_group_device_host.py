"""Device-resident grouped evaluation (b200dpf_group_eval_device) on the host: the symbol, the argument checks
that need no device, and the Python layers, which refuse wrong shapes, dtypes and device-resident bins before
the library is called.  No GPU needed."""
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


class _DeviceBins:
    """stands in for a CUDA tensor of bin ids, which a machine without a device cannot make"""
    is_cuda = True


def test_symbol_present():
    assert "b200dpf_group_eval_device" in B.SYMBOLS
    assert hasattr(C.CDLL(B.LIB_PATH), "b200dpf_group_eval_device")


def test_not_a_grouped_context_is_estate():
    bins = np.zeros(1, np.int32)
    assert B.lib().b200dpf_group_eval_device(None, C.c_void_p(16), bins, 1, B.PRF_AES128, C.c_void_p(16), None) == ESTATE
    assert "not a grouped context" in B.lib().b200dpf_last_error().decode()


def test_group_context_names_itself():
    ctx = B.GroupContext.__new__(B.GroupContext)    # no device: a context that was never created
    ctx.handle = C.c_void_p()
    with pytest.raises(B.B200DPFError, match=r"b200dpf_group_eval_device failed \(-4\).*not a grouped context"):
        ctx.eval_device(16, [0], B.PRF_AES128, 16)


def test_dpf_cpp_refuses_before_the_library():
    torch = pytest.importorskip("torch")
    import dpf
    cpp = dpf.dpf_cpp
    with pytest.raises(RuntimeError, match="group_eval_device: bins must be a contiguous CPU int32 tensor"):
        cpp.group_eval_device(16, torch.zeros(3, dtype=torch.int64), 3, [], B.PRF_AES128, 16, 0)
    with pytest.raises(RuntimeError, match="group_eval_device: bins must be a contiguous CPU int32 tensor"):
        cpp.group_eval_device(16, torch.zeros(3, dtype=torch.int32), 4, [], B.PRF_AES128, 16, 0)
    with pytest.raises(RuntimeError, match="group_eval_device: bins must be a contiguous CPU int32 tensor"):
        cpp.group_eval_device(16, torch.zeros((3, 2), dtype=torch.int32)[:, 0], 3, [], B.PRF_AES128, 16, 0)


def test_binned_dpf_refuses_before_the_library():
    """the refusals come first: a call that got past them would fail in dpf_cpp on the empty buffer list"""
    torch = pytest.importorskip("torch")
    import dpf
    d = dpf.BinnedDPF(prf=dpf.DPF.PRF_AES128)
    d.buffers = []
    d.table_effective_entry_size = 16
    keys = torch.zeros((3, 524), dtype=torch.int32)
    with pytest.raises(Exception, match=r"BinnedDPF\.eval_gpu_device: bins must be on the host.*synchronisation"):
        d.eval_gpu_device(keys, _DeviceBins())
    for bad in (keys, keys[:, :500], keys.long(), keys[0]):                    # host keys, wrong shape or dtype
        with pytest.raises(Exception, match=r"BinnedDPF\.eval_gpu_device: keys_dev must be a contiguous int32 \[B, 524\]"):
            d.eval_gpu_device(bad, [0, 0, 0])
    d.buffers = None
    with pytest.raises(Exception, match=r"BinnedDPF\.eval_gpu_device: keys_dev must be"):
        d.eval_gpu_device(keys, [0, 0, 0])
