"""Entries of up to 4096 columns on the host: the exact reference the GPU tests of wide entries use
(tests/wide_oracle.py, dot_u32_exact) against the column-by-column common.dot_u32, and the refusal of entry
sizes outside [1, 4096] by the plain and grouped create functions, which check the size before they open a
device.  No GPU needed."""
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
import wide_oracle as W  # noqa: E402
from common import dot_u32, random_table  # noqa: E402

EINVAL = -1
I32_MIN, I32_MAX = -2**31, 2**31 - 1


def shares_of(b, n, seed):
    return random_table(b, n, seed=seed)


@pytest.mark.parametrize("b,n,e", [(1, 1, 1), (3, 256, 63), (5, 256, 64), (2, 512, 65), (4, 300, 1000),
                                   (3, 128, 4096)])
def test_random_matches_dot_u32(b, n, e):
    s, t = shares_of(b, n, seed=n + e), random_table(n, e, seed=e)
    assert np.array_equal(W.dot_u32_exact(s, t), dot_u32(s, t))


def test_all_ones_at_2_20_rows():
    """(2^32 - 1)^2 = 1 mod 2^32 per row: the result is n; every limb sum is at its largest"""
    n = 1 << 20
    s = np.full((1, n), -1, np.int32)
    t = np.full((n, 2), -1, np.int32)
    got = W.dot_u32_exact(s, t)
    assert got.tolist() == [[n, n]]
    assert np.array_equal(got, dot_u32(s, t))
    # the same sum in row chunks that do not divide n
    assert np.array_equal(W.dot_u32_exact(s, t, row_chunk=(1 << 19) + 3), got)


def test_extreme_rows_and_shares():
    """INT32_MIN / INT32_MAX / -1 rows and shares, so every product and sum wraps"""
    n, e = 1024, 65
    t = random_table(n, e, seed=5)
    t[0], t[1], t[2], t[-3], t[-2], t[-1] = I32_MIN, I32_MAX, -1, I32_MAX, I32_MIN, -1
    t[:, 0], t[:, 31], t[:, -1] = I32_MIN, I32_MAX, -1
    s = shares_of(4, n, seed=6)
    s[0], s[1] = I32_MIN, I32_MAX
    s[2, ::2] = -1
    s[2, 1::2] = I32_MIN
    want = dot_u32(s, t)
    assert np.array_equal(W.dot_u32_exact(s, t), want)
    assert want[0, 0] == 0          # n * 2^62
    assert want[1, -1] == n         # n * -(2^31 - 1) = n * (2^31 + 1) mod 2^32


@pytest.mark.parametrize("row_chunk,col_chunk", [(1, 1), (100, 64), (256, 63), (257, 65), (1 << 20, 512)])
def test_chunks_straddled(row_chunk, col_chunk):
    """row and column counts that are and are not multiples of the chunk sizes"""
    for n, e in ((256, 64), (257, 130), (513, 65)):
        s, t = shares_of(3, n, seed=n), random_table(n, e, seed=e)
        assert np.array_equal(W.dot_u32_exact(s, t, row_chunk, col_chunk), dot_u32(s, t)), (n, e)


def test_one_dimensional_shares_and_bad_arguments():
    s, t = shares_of(1, 64, seed=1), random_table(64, 3, seed=2)
    assert np.array_equal(W.dot_u32_exact(s[0], t), dot_u32(s, t))
    with pytest.raises(ValueError, match="row_chunk"):
        W.dot_u32_exact(s, t, row_chunk=(1 << 20) + 1)
    with pytest.raises(ValueError, match="do not match"):
        W.dot_u32_exact(s, t[:63])


@pytest.mark.parametrize("suffix,n", [("", 2), ("_et", 8), ("_xor", 256)])
@pytest.mark.parametrize("e", [0, 4097, -1])
def test_create_refuses_entry_size(suffix, n, e):
    L = B.lib()
    table = np.zeros((1, 1), np.int32)         # refused before the table is read
    h = C.c_void_p()
    rc = getattr(L, "b200dpf_create" + suffix)(C.byref(h), table.ctypes.data_as(C.c_void_p), n, e, 0, 0, 1)
    assert not h
    assert rc == EINVAL
    assert L.b200dpf_last_error().decode() == "entry_size=%d out of range [1,4096]" % e


@pytest.mark.parametrize("e", [0, 4097, -1])
def test_group_create_refuses_entry_size(e):
    L = B.lib()
    tables = [np.zeros((1, 1), np.int32) for _ in range(2)]
    ptrs = (C.c_void_p * 2)(*[t.ctypes.data for t in tables])
    h = C.c_void_p()
    assert L.b200dpf_group_create(C.byref(h), ptrs, np.array([2, 64], np.int64), 2, e, 0) == EINVAL
    assert not h
    assert L.b200dpf_last_error().decode() == "entry_size=%d out of range [1,4096]" % e


@pytest.mark.parametrize("kw", [{}, {"early_termination": True}, {"xor": True}])
def test_python_context_refuses_4097_columns(kw):
    with pytest.raises(B.B200DPFError, match=r"entry_size=4097 out of range \[1,4096\]"):
        B.Context(np.zeros((256, 4097), np.int32), **kw)
    with pytest.raises(B.B200DPFError, match=r"entry_size=4097 out of range \[1,4096\]"):
        B.GroupContext([np.zeros((256, 4097), np.int32)], **kw)
