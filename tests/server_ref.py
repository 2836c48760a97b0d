"""Each server's exact answer on the bins of a grouped context, from the host share vectors -- TEST INFRASTRUCTURE ONLY.

The answer of one key on a bin of `rows` rows is

    out[e] = sum over r < rows of share[index(r)] * bin[r][e]   mod 2^32
    out[e] = XOR over r < rows of (share[index(r)] ? bin[r][e] : 0)          (XOR-shared keys)

with index(r) = trimmed_alpha(r, rows) on a trimmed bin and r on a bin of a power-of-two size, and `share` the key's
host evaluation over its whole domain (b200dpf_eval_cpu, _et, _xor; tests/plan_matrix.py and tests/wide_oracle.py
anchor those to the per-index oracles).  Nothing here runs on a GPU.  A random key weights every row of its bin by a
pseudo-random share, so one exact comparison covers the whole bin: a row dropped, counted twice, read from a neighbour
or written where it does not belong changes the answer of both servers alike, which their difference cannot see.

The keys evaluate on host threads (ctypes releases the GIL while b200dpf_eval_cpu runs)."""
import functools
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402
import wide_oracle  # noqa: E402
import xor_oracle  # noqa: E402

SUFFIX = {"standard": "", "et": "_et", "xor": "_xor"}
NTHREADS = min(16, os.cpu_count() or 1)


def domain(rows, kind, trimmed=True):
    """the n of the keys a bin of `rows` rows takes"""
    return B.trimmed_domain(rows, SUFFIX[kind]) if trimmed else rows


@functools.lru_cache(maxsize=None)
def key_index(rows, kind, trimmed=True):
    """int64 [rows]: the key index of every row of a bin"""
    if not trimmed:
        return np.arange(rows, dtype=np.int64)
    return np.array([B.trimmed_alpha(r, rows, SUFFIX[kind]) for r in range(rows)], np.int64)


def shares(kind, prf, keys):
    """the host share vectors of `keys` (int32 [K, 524], one domain): int32 [K, n], or uint8 share bits for XOR-shared keys"""
    keys = np.ascontiguousarray(keys, np.int32).reshape(-1, B.KEY_WORDS)
    ev = {"standard": B.eval_cpu, "et": B.eval_cpu_et, "xor": B.eval_cpu_xor}[kind]
    with ThreadPoolExecutor(NTHREADS) as ex:
        out = list(ex.map(lambda k: ev(k, prf), keys))
    if kind == "xor":
        return np.stack([xor_oracle.unpack_bits(w) for w in out])
    return np.stack(out)


def bin_answers(kind, prf, keys, table, trimmed=True):
    """int32 [K, E]: each server's answer of `keys` (all for this bin) on the bin `table` (int32 [rows, E])"""
    keys = np.ascontiguousarray(keys, np.int32).reshape(-1, B.KEY_WORDS)
    table = np.ascontiguousarray(table, np.int32)
    if keys.shape[0] == 0:
        return np.zeros((0, table.shape[1]), np.int32)
    sh = shares(kind, prf, keys)
    assert sh.shape[1] == domain(table.shape[0], kind, trimmed), "keys of another domain"
    return weigh(kind, sh, table, trimmed)


def weigh(kind, sh, table, trimmed=True):
    """the answers from share vectors sh [K, n] of keys for the bin `table`"""
    sel = sh[:, key_index(table.shape[0], kind, trimmed)]
    if kind == "xor":
        return xor_oracle.xor_rows(sel, table)
    return wide_oracle.dot_u32_exact(sel, table)


def grouped_answers(kind, prf, keys, bins, tables, trimmed=True):
    """int32 [K, E]: the answer of key j on bin bins[j] of `tables`; a key whose bin is out of range answers zeros"""
    keys = np.ascontiguousarray(keys, np.int32).reshape(-1, B.KEY_WORDS)
    bins = np.asarray(bins, np.int64)
    out = np.zeros((keys.shape[0], tables[0].shape[1]), np.int32)
    valid = (bins >= 0) & (bins < len(tables))
    by_rows = {}
    for g in np.unique(bins[valid]):
        by_rows.setdefault(tables[g].shape[0], []).append(int(g))
    for rows, group in by_rows.items():       # one host evaluation per key, the bins of one size together
        at = np.flatnonzero(np.isin(bins, group))
        sh = shares(kind, prf, keys[at])
        for g in group:
            mine = bins[at] == g
            out[at[mine]] = weigh(kind, sh[mine], tables[g], trimmed)
    return out


def query_answers(kind, prf, keys, tables, trimmed=True):
    """int32 [Q, nbins, E]: the answers of queries of one key per bin (int32 [Q, nbins, 524], key g for bin g)"""
    keys = np.ascontiguousarray(keys, np.int32)
    nq, nbins = keys.shape[:2]
    bins = np.tile(np.arange(nbins), nq)
    return grouped_answers(kind, prf, keys.reshape(-1, B.KEY_WORDS), bins, tables, trimmed).reshape(nq, nbins, -1)


def unpack_queries(kind, bin_rows, packed, trimmed=True):
    """compact queries uint8 [Q, query_bytes] (each query its keys' key_pack forms back to back) -> int32
    [Q, nbins, 524] wire-format keys"""
    s = SUFFIX[kind]
    lane_bits = B.KINDS[s][0]
    sizes = [B.lib().b200dpf_key_packed_size(domain(r, kind, trimmed).bit_length() - 1 - lane_bits) for r in bin_rows]
    packed = np.ascontiguousarray(packed, np.uint8)
    assert packed.shape[1] == sum(sizes)
    unpack = getattr(B, "key_unpack" + s)
    out = np.zeros((packed.shape[0], len(bin_rows), B.KEY_WORDS), np.int32)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    for q in range(packed.shape[0]):
        for g in range(len(bin_rows)):
            out[q, g] = unpack(packed[q, offs[g]:offs[g + 1]].tobytes())
    return out


def edge_rows(rows, kind, trimmed=True):
    """rows of a bin to select: the first, the last, and those whose key indices are nearest 0101.. and 1010.. (paths
    that turn at every level, so that the rows off the path lie on both sides of it at every level)"""
    idx = key_index(rows, kind, trimmed)
    n = domain(rows, kind, trimmed)
    out = [0, rows - 1]
    for pattern in (0x5555555555555555, 0xAAAAAAAAAAAAAAAA):
        out.append(int(np.argmin(np.abs(idx - (pattern & (n - 1))))))
    return out
