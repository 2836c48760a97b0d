"""Argument checks of the row-update API that need no GPU: the Python layers refuse bad calls before
anything reaches the extension, and the C ABI rejects a null context."""
import ctypes as C

import numpy as np
import pytest
import torch

import b200dpf


def test_update_before_eval_init():
    import dpf
    from sharded import ShardedDPF
    with pytest.raises(Exception, match="Must call `eval_init`"):
        dpf.DPF().update_rows([0], torch.zeros((1, 16), dtype=torch.int32))
    with pytest.raises(Exception, match="Must call `eval_init`"):
        dpf.BinnedDPF().update_rows([0], [0], torch.zeros((1, 16), dtype=torch.int32))
    with pytest.raises(Exception, match="Must call `eval_init`"):
        ShardedDPF(prf=3).update_rows([0], torch.zeros((1, 16), dtype=torch.int32))


def test_update_shape_and_dtype_errors():
    """Checked in Python: the fake buffer handle below would make any extension call fail differently."""
    import dpf
    d = dpf.DPF()
    d.buffers = [None]
    d.table_effective_entry_size, d.table_rows = 4, 128
    rows = torch.zeros((2, 4), dtype=torch.int32)
    with pytest.raises(Exception, match="indices must be a 1-D integer"):
        d.update_rows(torch.tensor([0.0, 1.0]), rows)
    with pytest.raises(Exception, match="indices must be a 1-D integer"):
        d.update_rows(torch.tensor([[0, 1]]), rows)
    with pytest.raises(Exception, match=r"rows must be \[2, 4\]"):
        d.update_rows([0, 1], torch.zeros((2, 5), dtype=torch.int32))
    with pytest.raises(Exception, match=r"rows must be \[3, 4\]"):
        d.update_rows([0, 1, 2], rows)
    with pytest.raises(Exception, match="real-valued"):
        d.update_rows([0, 1], rows.bool())
    with pytest.raises(Exception, match=r"out of range \[0, 128\)"):
        d.update_rows([0, 128], rows)
    with pytest.raises(Exception, match=r"out of range \[0, 128\)"):
        d.update_rows([-1, 3], rows)
    b = dpf.BinnedDPF()
    b.buffers = [None]
    b.table_effective_entry_size = 4
    with pytest.raises(Exception, match="one bin per index"):
        b.update_rows([0], [0, 1], rows)
    with pytest.raises(Exception, match="one bin per index"):
        b.update_rows([0.5, 1.0], [0, 1], rows)


def test_update_abi_null_context():
    L = b200dpf.lib()
    idx = np.array([0], np.int64)
    rows = np.zeros((1, 16), np.int32)
    assert L.b200dpf_update_rows(None, idx, rows, 1) == -1
    assert b"null context" in L.b200dpf_last_error()
    assert L.b200dpf_update_rows_device(None, C.c_void_p(0), C.c_void_p(0), 1, None) == -1
    assert b"null context" in L.b200dpf_last_error()
    assert L.b200dpf_group_update_rows(None, np.zeros(1, np.int32), idx, rows, 1) == -1
    assert b"null context" in L.b200dpf_last_error()
