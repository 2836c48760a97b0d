"""The option matrix of tests/test_gpu_plan_matrix.py, without a device: its rows cover every pair of levels
of every two options, are the same on every call, and set only values b200dpf_ctx_set_option accepts."""
import itertools
import os
import re

import pytest

import plan_matrix as PM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# kKnobs (gpu-dpf_b200/csrc/dpf_capi.cu): option -> (default, lowest, highest accepted value).  A copy, so the
# ranges are checked without a context, which needs a device; test_knob_table_copy keeps it in step.
KNOBS = {
    "leaf_cache": (1, 0, 1),
    "leaf_cache_mb": (16384, 1, 1 << 20),
    "lane_split": (1, 0, 1),
    "frontier": (1, 0, 1),
    "frontier_mb": (256, 1, 1 << 16),
    "subtree_log2": (0, 0, 16),
    "mac_tma": (1, 0, 1),
    "one_launch": (1, 0, 1),
    "balance_top": (1, 0, 1),
    "timing": (0, 0, 1),
    "top_log2": (0, 0, 7),
    "tma_rows": (0, 0, 1),
}


def _expr(text):
    return int(eval(text, {"__builtins__": {}}))    # the table's bounds are literals and shifts of literals


def test_knob_table_copy():
    src = open(os.path.join(ROOT, "gpu-dpf_b200", "csrc", "dpf_capi.cu")).read()
    table = src[src.index("constexpr KnobInfo kKnobs[]"):]
    table = table[:table.index("};")]
    rows = re.findall(r'\{&Kn::(\w+),\s*([^,]+),\s*"\w+",\s*"(\w+)",\s*([^,]+),\s*([^}]+)\}', table)
    assert rows, "kKnobs not found"
    got = {}
    for field, dflt, name, lo, hi in rows:
        assert field == name
        got[name] = (_expr(dflt), _expr(lo), _expr(hi))
    assert got == KNOBS


def test_every_option_is_in_the_matrix():
    assert set(PM.OPTIONS) == set(KNOBS)
    for name, levels in PM.OPTIONS.items():
        dflt, lo, hi = KNOBS[name]
        assert levels[0] == dflt, name
        assert len(set(levels)) == len(levels), name
        assert lo in levels, name
        for v in levels:
            assert lo <= v <= hi, (name, v)


@pytest.mark.parametrize("seed", (0, 1))
def test_rows_cover_every_pair(seed):
    rows = PM.pairwise_rows(seed)
    assert rows[0] == PM.DEFAULTS
    assert 16 <= len(rows) <= 30, len(rows)      # at least 4 x 4 for subtree_log2 x top_log2
    for row in rows:
        assert set(row) == set(PM.OPTIONS)
        for name, v in row.items():
            assert v in PM.OPTIONS[name], (name, v)
            assert KNOBS[name][1] <= v <= KNOBS[name][2], (name, v)
    for a, b in itertools.combinations(PM.OPTIONS, 2):
        seen = {(row[a], row[b]) for row in rows}
        for va in PM.OPTIONS[a]:
            for vb in PM.OPTIONS[b]:
                assert (va, vb) in seen, (a, va, b, vb)


def test_rows_are_deterministic():
    assert PM.pairwise_rows(0) == PM.pairwise_rows(0)
    assert PM.pairwise_rows(3) == PM.pairwise_rows(3)


def test_combine_and_reconstruct():
    import numpy as np
    a = np.array([[0x7fffffff, -1]], np.int32)
    b = np.array([[1, -1]], np.int32)
    assert PM.combine("standard", [a, b]).tolist() == [[-2**31, -2]]
    assert PM.combine("xor", [a, b]).tolist() == [[0x7ffffffe, 0]]
    assert PM.reconstruct("et", a, b).tolist() == [[0x7ffffffe, 0]]
    assert PM.reconstruct("xor", a, b).tolist() == [[0x7ffffffe, 0]]
