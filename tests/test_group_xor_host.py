"""Grouped (batch-PIR) contexts for XOR-shared keys on the host: the argument checks of
b200dpf_group_create_xor, which refuse a bad bin list before any device is touched, and the Python
surfaces.  No GPU needed."""
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

EINVAL = -1


def create_xor(sizes, entry_size=16, nbins=None):
    """b200dpf_group_create_xor with the given row counts -> (rc, error text).  The sizes are refused
    before a table is read, so each table is one row."""
    L = B.lib()
    tables = [np.zeros((1, max(entry_size, 1)), np.int32) for _ in sizes]
    ptrs = (C.c_void_p * max(len(tables), 1))(*[t.ctypes.data for t in tables])
    h = C.c_void_p()
    rc = L.b200dpf_group_create_xor(C.byref(h), ptrs, np.array(list(sizes) or [0], np.int64),
                                    len(tables) if nbins is None else nbins, entry_size, 0)
    if h:
        L.b200dpf_destroy(h)
    return rc, L.b200dpf_last_error().decode()


def test_symbol_present():
    assert "b200dpf_group_create_xor" in B.SYMBOLS
    assert hasattr(C.CDLL(B.LIB_PATH), "b200dpf_group_create_xor")


@pytest.mark.parametrize("sizes,what", [
    ([128], "n=128"),             # one leaf of 128 rows: below the smallest tree (two leaves)
    ([256, 128], "n=128"),
    ([256, 2], "n=2"),            # a size the standard grouped context accepts
    ([24], "n=24"),               # not a power of two
    ([256, 1000], "n=1000"),
    ([256, 1 << 32], "n=4294967296"),
])
def test_bad_bin_size_is_einval(sizes, what):
    rc, err = create_xor(sizes)
    assert rc == EINVAL, err
    assert what in err and "[256, 2^31]" in err


def test_bad_bin_list_and_entry_size_are_einval():
    rc, err = create_xor([256], nbins=0)
    assert rc == EINVAL and "nbins=0" in err
    for e in (0, 4097):
        rc, err = create_xor([256], entry_size=e)
        assert rc == EINVAL and "entry_size=%d" % e in err
    h = C.c_void_p()
    sizes = np.array([256], np.int64)
    assert B.lib().b200dpf_group_create_xor(C.byref(h), None, sizes, 1, 16, 0) == EINVAL
    assert B.lib().b200dpf_group_create_xor(None, None, sizes, 1, 16, 0) == EINVAL


def test_python_surfaces():
    """each entry point fails loudly and names itself (a 128-row bin is refused with or without a device)"""
    with pytest.raises(ValueError, match="one kind of key"):
        B.GroupContext([np.zeros((256, 16), np.int32)], xor=True, early_termination=True)
    with pytest.raises(B.B200DPFError, match="b200dpf_group_create_xor"):
        B.GroupContext([np.zeros((128, 16), np.int32)], xor=True)
    torch = pytest.importorskip("torch")
    import dpf
    with pytest.raises(Exception, match=r"dpf_cpp\.group_init_xor or b200dpf\.GroupContext\(xor=True\)"):
        dpf.BinnedDPF(xor=True)
    with pytest.raises(RuntimeError, match="group_init_xor"):
        dpf.dpf_cpp.group_init_xor([torch.zeros((128, 16), dtype=torch.int32)])
