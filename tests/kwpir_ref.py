"""The keyword-PIR layout restated in numpy from include/b200dpf.h (b200dpf_kwpir_*): the hash h_c, the round-based
cuckoo placement, the tags it leaves in the three bins and the bins' whole contents.  Shared by the host and the GPU
tests."""
import numpy as np

M64 = (1 << 64) - 1
GOLDEN = np.uint64(0x9E3779B97F4A7C15)
MAX_ROUNDS = 1024


def mix(z):
    """the SplitMix64 finalizer on a uint64 array"""
    z = np.asarray(z, np.uint64)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
    return z ^ (z >> np.uint64(31))


def h(c, w, m, seed):
    """h_c(w) = ((mix(mix(w ^ seed) ^ ((c + 1) * 0x9E3779B97F4A7C15)) >> 32) * m) >> 32, mod 2^64"""
    with np.errstate(over="ignore"):
        z = mix(mix(np.asarray(w, np.uint64) ^ np.uint64(seed & M64)) ^ (np.uint64(c + 1) * GOLDEN))
        return (((z >> np.uint64(32)) * np.uint64(m)) >> np.uint64(32)).astype(np.int64)


def rows3(keywords, m, seed):
    """[Q, 3]: the in-bin row of each keyword in bins 0, 1, 2"""
    return np.stack([h(c, keywords, m, seed) for c in range(3)], axis=1)


def place(keywords, m, seed, max_rounds=MAX_ROUNDS):
    """The placement rule: (rounds, owner) with owner int64 [3 * m] (slot c * m + row -> item index, -1 empty), or
    (None, owner) when items are still homeless after max_rounds rounds."""
    keywords = np.asarray(keywords, np.uint64)
    n = len(keywords)
    cand = np.stack([c * m + h(c, keywords, m, seed) for c in range(3)])        # [3, n] slots
    owner = np.full(3 * m, -1, np.int64)
    choice = np.zeros(n, np.int64)
    homeless = np.arange(n)
    for r in range(max_rounds):
        if len(homeless) == 0:
            return r, owner
        slot = cand[choice[homeless], homeless]
        bid = np.full(3 * m, n, np.int64)
        np.minimum.at(bid, slot, homeless)                   # each slot's smallest bidding index wins
        win = bid[slot] == homeless
        old = owner[slot[win]]
        owner[slot[win]] = homeless[win]
        nxt = np.concatenate([old[old >= 0], homeless[~win]])  # evicted owners and losing bidders
        choice[nxt] = (choice[nxt] + 1) % 3
        homeless = nxt
    return (max_rounds if len(homeless) == 0 else None), owner


def tags(keywords, owner, m):
    """uint64 [3, m]: keyword + 1 of each slot's item, 0 for an empty slot"""
    keywords = np.asarray(keywords, np.uint64)
    out = np.zeros(3 * m, np.uint64)
    full = owner >= 0
    with np.errstate(over="ignore"):
        out[full] = keywords[owner[full]] + np.uint64(1)
    return out.reshape(3, m)


def bins(keywords, values, m, seed):
    """The contents of the three bins: int32 [m, E + 2] each.  The slot of an item holds its value in columns 0 .. E-1
    and its tag w + 1 in columns E (low 32 bits) and E + 1 (high 32 bits); an empty slot is all zeros.  The slots are
    those of place(); a placement that does not finish raises."""
    values = np.asarray(values, np.int32)
    rounds, owner = place(keywords, m, seed)
    if rounds is None:
        raise ValueError("the placement of %d items in 3 x %d slots does not finish under seed %d" % (len(values), m, seed))
    e = values.shape[1]
    out = np.zeros((3 * m, e + 2), np.int32)
    full = owner >= 0
    out[full, :e] = values[owner[full]]
    tag = tags(keywords, owner, m).reshape(-1)
    out[:, e] = (tag & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.int32)
    out[:, e + 1] = (tag >> np.uint64(32)).astype(np.uint32).view(np.int32)
    return [out[c * m:(c + 1) * m] for c in range(3)]


def default_m(n, expansion=1.3):
    return max(-(-n // 3), int(np.ceil(expansion * n / 3)))
