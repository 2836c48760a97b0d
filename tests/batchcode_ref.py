"""The batch-code layout restated in numpy from include/b200dpf.h (b200dpf_batchcode_*): the SplitMix64 finalizer, copy
c's Feistel network and its cycle-walked permutation pi_c, and the bins they fill.  Shared by the host and the GPU
tests; only `locate` asks the library."""
import numpy as np

M64 = (1 << 64) - 1
COPIES = 3


def mix(z):
    """the SplitMix64 finalizer on a uint64 array"""
    z = np.asarray(z, np.uint64)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
    return z ^ (z >> np.uint64(31))


def half_bits(n):
    h = 1
    while (1 << (2 * h)) < n:
        h += 1
    return h


def feistel(seed, c, x, h):
    mask = np.uint64((1 << h) - 1)
    l, r = x >> np.uint64(h), x & mask
    for i in range(4):
        f = mix(np.uint64(seed) ^ mix((np.uint64(c * 8 + i) << np.uint64(32)) | r)) & mask
        l, r = r, l ^ f
    return (l << np.uint64(h)) | r


def perm(n, seed, c, rows):
    """pi_c of every row in `rows`: the Feistel network, cycle-walked below n"""
    h = half_bits(n)
    x = feistel(seed, c, np.asarray(rows, np.uint64), h)
    while True:
        out = x >= np.uint64(n)
        if not out.any():
            return x.astype(np.int64)
        x[out] = feistel(seed, c, x[out], h)


def per_copy(n, nbins, j):
    """m_j: the rows of one copy in bin j"""
    return (n - j + nbins - 1) // nbins


def locate(n, nbins, seed, row):
    """the library's answer (b200dpf_batchcode_locate): ([bin of copy c], [in-bin row of copy c]) for c = 0, 1, 2"""
    import b200dpf as B
    bins, rows = B.batchcode_locate(n, nbins, seed, row)
    return [int(b) for b in bins], [int(r) for r in rows]


def bins(table, n, nbins, seed):
    """The contents of every bin: a list of nbins int32 arrays [3 m_j, E].  Copy c of table row r, with x = pi_c(r),
    is row c * m_j + floor(x / nbins) of bin j = x mod nbins."""
    table = np.asarray(table, np.int32)
    assert table.shape[0] == n
    m = np.array([per_copy(n, nbins, j) for j in range(nbins)], np.int64)
    out = [np.zeros((COPIES * int(m[j]), table.shape[1]), np.int32) for j in range(nbins)]
    filled = [np.zeros(COPIES * int(m[j]), np.int32) for j in range(nbins)]
    rows = np.arange(n)
    for c in range(COPIES):
        x = perm(n, seed, c, rows)
        j, q = x % nbins, x // nbins
        for b in np.unique(j):
            sel = j == b
            at = c * m[b] + q[sel]
            out[b][at] = table[sel]
            filled[b][at] += 1
    assert all((f == 1).all() for f in filled), "the restated layout does not fill every bin row exactly once"
    return out
