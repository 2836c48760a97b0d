/*
 * dpf_kernels.cuh -- launch interface between the C-ABI layer (dpf_capi.cu)
 * and the sm_90a kernels (dpf_kernels.cu).  Plain structs, no torch.
 */
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "dpf_core.cuh"

namespace b200dpf {

/* RowPlacement::depth of a trimmed table or bin, which keeps the caller's row order */
enum { PLACE_IDENTITY = -1 };

/* Where the rows of one table live in the device table of its context: a whole table, one shard of one (an entry
 * range, DESIGN.md section 5) or one bin of a grouped context.  Table creation, row updates and the key generator all
 * read it from here.  Natural row i is row i & (2^lane_bits - 1) of leaf v = i >> lane_bits; a leaf's rows stay
 * adjacent.
 *   owns(i)        0 <= i < n and (v & own_mask) == own_val.  Shard r of G = 2^shift owns the leaves under tree node r
 *                  of level `shift`, those with bitrev(v mod G, shift) = r (own_mask = G - 1, own_val = bitrev(r, shift));
 *                  any other placement has no shards (mask, value and shift 0).
 *   device_row(i)  first + (bitrev(v >> shift, depth) << lane_bits | (i & (2^lane_bits - 1))): breadth-first leaf order
 *                  over the depth leaf levels below the shard's root, the order the evaluation kernels walk the tree in.
 *                  A trimmed table or bin (depth = PLACE_IDENTITY) stores row i at device row first + i.
 *   natural_row(q) the natural row held by device row first + q, the inverse of device_row. */
struct RowPlacement {
    uint64_t first;           /* first device row */
    uint32_t n;               /* live rows: natural rows [0, n) */
    int lane_bits;            /* log2 rows per leaf: 0, 2 (early-terminated keys) or 7 (XOR-shared keys) */
    int depth;                /* width of the leaf bit reversal, or PLACE_IDENTITY */
    uint32_t own_mask, own_val;
    int shift;                /* log2 shards */

    DPF_HD bool owns(int64_t i) const
    {
        return i >= 0 && i < (int64_t)n && ((uint32_t)(i >> lane_bits) & own_mask) == own_val;
    }
    DPF_HD uint64_t device_row(int64_t i) const
    {
        if (depth == PLACE_IDENTITY) return first + (uint64_t)i;
        const uint32_t leaf = bitrev((uint32_t)(i >> lane_bits) >> shift, depth);
        return first + (((uint64_t)leaf << lane_bits) | ((uint32_t)i & ((1u << lane_bits) - 1u)));
    }
    DPF_HD int64_t natural_row(uint64_t q) const
    {
        if (depth == PLACE_IDENTITY) return (int64_t)q;
        const uint32_t leaf = bitrev((uint32_t)(q >> lane_bits), depth) << shift | own_val;
        return ((int64_t)leaf << lane_bits) | (int64_t)(q & ((1u << lane_bits) - 1u));
    }
};

/* The key index of row r of a trimmed table whose tree has `depth` leaf levels (b200dpf_trimmed_alpha): r sits at leaf
 * position r >> lane_bits, which the key reaches as leaf bitrev(r >> lane_bits, depth). */
DPF_HD uint64_t trimmed_alpha(uint64_t r, int depth, int lane_bits)
{
    return ((uint64_t)bitrev((uint32_t)(r >> lane_bits), depth) << lane_bits) | (r & ((1u << lane_bits) - 1u));
}

/* Batch-code layout (b200dpf_batchcode_create, DESIGN.md section 13): every row of an n-row table has three copies in
 * nbins trimmed bins, each copy placed by its own keyed permutation of [0, n).  Table creation, row updates, the host
 * planner and the device planner all place rows through this one definition; include/b200dpf.h states it in full. */
enum { BATCHCODE_COPIES = 3, BATCHCODE_ROUNDS = 4, BATCHCODE_MAX_K = 4096 };

/* The SplitMix64 finalizer */
DPF_HD uint64_t batchcode_mix(uint64_t z)
{
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

struct BatchCodeLayout {
    uint64_t n;               /* rows of the table, [1, 2^31] */
    uint64_t seed;            /* the public layout seed */
    uint32_t nbins;           /* B, [1, min(n, 2^20)] */
    int half;                 /* h: the Feistel network is over 2h >= max(2, ceil(log2 n)) bits */

    /* One pass of the balanced Feistel network of copy c over [0, 2^2h): x = (L, R) of h bits each, and each round
     * maps (L, R) to (R, L ^ F(round, R)) with F(i, R) = mix(seed ^ mix((c * 8 + i) << 32 | R)) mod 2^h. */
    DPF_HD uint64_t feistel(int copy, uint64_t x) const
    {
        const uint64_t mask = ((uint64_t)1 << half) - 1;
        uint64_t l = x >> half, r = x & mask;
        for (int round = 0; round < BATCHCODE_ROUNDS; round++) {
            const uint64_t f = batchcode_mix(seed ^ batchcode_mix((uint64_t)(copy * 8 + round) << 32 | r)) & mask;
            const uint64_t t = l ^ f;
            l = r;
            r = t;
        }
        return l << half | r;
    }
    /* pi_c(r): the Feistel network applied until the value is below n (cycle walking), a permutation of [0, n) */
    DPF_HD uint64_t perm(int copy, uint64_t r) const
    {
        uint64_t x = r;
        do x = feistel(copy, x); while (x >= n);
        return x;
    }
    /* m_j: the x in [0, n) with x mod B = j.  Bin j holds 3 m_j rows. */
    DPF_HD uint64_t per_copy(uint32_t j) const { return (n - j + nbins - 1) / nbins; }
    DPF_HD uint32_t bin_of(int copy, uint64_t r) const { return (uint32_t)(perm(copy, r) % nbins); }
    /* copy c of row r: bin x mod B, row c m_j + x / B of that bin, for x = pi_c(r) */
    DPF_HD void locate(int copy, uint64_t r, uint32_t *bin, uint64_t *row) const
    {
        const uint64_t x = perm(copy, r);
        *bin = (uint32_t)(x % nbins);
        *row = (uint64_t)copy * per_copy(*bin) + x / nbins;
    }
};

/*
 * The plan of one query of k wanted rows (b200dpf_batchcode_plan): Kuhn's augmenting paths over the wanted rows in
 * order, trying copies 0, 1, 2 in order, a row that repeats a placed earlier row sharing its bin.  Rows outside
 * [0, n) are not placed.  It runs in the caller's outputs: while the matching is built, state[v] (v < nbins) holds
 * the wanted row matched to bin v plus one (bits 0..15, 0 for none), that row's copy (bits 16..17) and the root of
 * the last search that visited v plus one (bits 32..47); slots[u] holds the row and copy (plus one, and in bits
 * 16..17) a search came from to reach row u.  At the end state becomes the alphas (bin v's in-bin row to query, 0
 * for a bin no row uses) and slots the bin answering each wanted row, or -1.  The host and the device run this same
 * code, so their plans agree bit for bit.
 */
DPF_HD void batchcode_plan_query(const BatchCodeLayout &L, const int64_t *wanted, int k, int64_t *state, int32_t *slots)
{
    const int64_t n = (int64_t)L.n;
    for (uint32_t v = 0; v < L.nbins; v++) state[v] = 0;
    for (int i = 0; i < k; i++) {
        const int64_t r = wanted[i];
        if (r < 0 || r >= n) continue;
        bool placed = false;        /* an earlier occurrence of r holds one of r's bins */
        for (int c = 0; c < BATCHCODE_COPIES; c++) {
            const int m = (int)(state[L.bin_of(c, (uint64_t)r)] & 0xffff);
            placed |= m != 0 && wanted[m - 1] == r;
        }
        if (placed) continue;       /* (an earlier occurrence that was not placed fails again: no augmenting path appears) */
        const int64_t stamp = (int64_t)(i + 1) << 32;
        int u = i, c = 0;
        for (;;) {
            if (c == BATCHCODE_COPIES) {              /* row u has no way out: back to the row that reached it */
                if (u == i) break;
                const int32_t p = slots[u];
                u = (p & 0xffff) - 1;
                c = (p >> 16) + 1;
                continue;
            }
            const uint32_t v = L.bin_of(c, (uint64_t)wanted[u]);
            const int64_t s = state[v];
            if ((s & ((int64_t)0xffff << 32)) == stamp) {
                c++;
                continue;
            }
            state[v] = (s & 0xffffffff) | stamp;
            const int w = (int)(s & 0xffff) - 1;
            if (w >= 0) {                              /* bin v is taken: try to move its row w */
                slots[w] = (u + 1) | (c << 16);
                u = w;
                c = 0;
                continue;
            }
            for (;;) {                                 /* an augmenting path: every row on it takes the bin it tried */
                const uint32_t b = L.bin_of(c, (uint64_t)wanted[u]);
                state[b] = (state[b] & ~(int64_t)0xffffffff) | (int64_t)((u + 1) | (c << 16));
                if (u == i) break;
                const int32_t p = slots[u];
                u = (p & 0xffff) - 1;
                c = p >> 16;
            }
            break;
        }
    }
    for (int i = 0; i < k; i++) {
        const int64_t r = wanted[i];
        int32_t slot = -1;
        for (int c = 0; r >= 0 && r < n && c < BATCHCODE_COPIES && slot < 0; c++) {
            const uint32_t v = L.bin_of(c, (uint64_t)r);
            const int m = (int)(state[v] & 0xffff);
            if (m != 0 && wanted[m - 1] == r) slot = (int32_t)v;
        }
        slots[i] = slot;
    }
    for (uint32_t v = 0; v < L.nbins; v++) {
        const int m = (int)(state[v] & 0xffff);
        const int c = (int)((state[v] >> 16) & 3);
        state[v] = m == 0 ? 0 : (int64_t)((uint64_t)c * L.per_copy(v) + L.perm(c, (uint64_t)wanted[m - 1]) / L.nbins);
    }
}

/* Keyword-PIR layout (b200dpf_kwpir_create, DESIGN.md section 14): n (keyword, value) items in a cuckoo hash table of
 * three tables (bins) of m slots; an item sits in one of its three candidate slots, its row the value then the tag
 * w + 1 in two columns.  Table creation, row updates and both locators place keywords through this one definition;
 * include/b200dpf.h states it in full. */
enum { KWPIR_TABLES = 3, KWPIR_MAX_ROUNDS = 1024, KWPIR_MAX_VALUE = 4094 };

struct KeywordLayout {
    uint64_t n;               /* items, [1, 2^30] */
    uint64_t m;               /* slots per table, [ceil(n / 3), 2^31] */
    uint64_t seed;            /* the public layout seed */
    int value_size;           /* E: value columns; the tag is columns E and E + 1 */

    /* h_c(w): keyword w's candidate row in table c, ((mix(mix(w ^ seed) ^ (c + 1) * golden) >> 32) * m) >> 32.
     * The product is below 2^63 because m <= 2^31. */
    DPF_HD uint64_t row(int c, uint64_t w) const
    {
        const uint64_t z = batchcode_mix(batchcode_mix(w ^ seed) ^ ((uint64_t)(c + 1) * 0x9E3779B97F4A7C15ull));
        return ((z >> 32) * m) >> 32;
    }
};

/* One traversal phase of a launch: which subtrees the work items are, where an item starts and
 * which ticket counters hand the items out. */
struct PhaseParams {
    int s;                    /* log2 leaves per work item (one warp = 32 keys x 2^s)   */
    /* where a work item starts: the key's root seed, or a node of a precomputed
     * frontier (seeds of every depth-F node of this shard)                            */
    const uint4 *frontier_in; /* [key_groups][nfront][kpw keys] or null                 */
    int front_shift;          /* work item q starts at frontier node q >> front_shift   */
    int walk_first_level;     /* correction-word level of the first walk step           */
    int walk_steps;           /* walk steps from the start node to the subtree root     */
    int level_base;           /* level of the subtree's bottom expansion (0 = leaves)   */
    uint32_t sub_first;       /* breadth-first index of the shard's first 2^s-subtree   */
    uint32_t nsub;            /* number of 2^s-subtrees issued in this shard: all of them, or on
                                 a trimmed context those over its padded table rows        */
    uint32_t *counters;       /* [key_groups] tickets, zero at phase start; one ticket =
                                 32/kpw consecutive subtrees for the group's kpw keys   */
    int stack_split;          /* pending-sibling stack levels [0, split) live in the lo
                                 region, the rest in the hi region                      */
};

/* Grouped evaluation (batch PIR: many small tables -- "bins" -- behind one context, one launch for a
 * mixed list of (bin, key) pairs): a key group is <= 32 keys of the SAME bin, so its warp still
 * walks one tree shape and shares each table row.  One descriptor per key group. */
struct GroupDesc {
    uint32_t key_first;       /* first key of the group in the (bin-sorted) key array       */
    uint32_t nkeys;           /* 1..32                                                      */
    int32_t depth;            /* log2 of the bin's table size (MODE_GROUPED_ET, _XOR: of its leaves) */
    int32_t s;                /* log2 leaves per work item for this group                   */
    uint32_t nsub;            /* work items (2^s-leaf subtrees): 2^(depth - s), or on a trimmed
                                 context those over the bin's padded rows                   */
    uint32_t pad;
    uint64_t table_off_v;     /* bin's first row, in uint4 units from EvalParams::table     */
};

/* What a block of a mode that draws work units (ModeTraits::units) takes in one draw: work items
 * [first, first + count) of key group `group`.  The host lists them in group-major order. */
struct WorkUnit {
    uint32_t group, first, count, pad;
};

/* Parameters of one evaluation launch (one pass over <= 16*NVMAX columns). */
struct EvalParams {
    const uint4 *keys;        /* [nkeys] keys, key_stride_v 128-bit slots apart          */
    uint32_t key_stride_v;    /* reference wire format: 131; compact: 2 + 4*depth        */
    uint32_t key_root_v;      /* slot of the root seed: 129 (reference) / 1 (compact)    */
    int key_compact;          /* 0: cw_1 at slots 1.., cw_2 at 65.. (dpf_wrapper.cu:26-46);
                                 1: slot 2 + 4*level + 2*bank + bit                      */
    int nkeys;
    int kpw_log2;             /* log2 keys per warp (5 = one key per lane).  With fewer
                                 keys than lanes the spare lanes take further subtrees of
                                 the same keys: lane = (key = lane % kpw, subtree slot =
                                 lane / kpw), so small batches still fill the warp       */
    int key_groups;           /* ceil(nkeys / kpw)                                       */
    const uint4 *table;       /* this shard's rows in breadth-first leaf order          */
    uint32_t row_stride_v;    /* uint4 per table row (padded entry size / 4)            */
    uint32_t col_off_v;       /* first uint4 column of this pass                        */
    uint32_t *out;            /* [nkeys][out_stride] uint32, zero before the main phase  */
    uint32_t out_stride;
    uint32_t col_off;         /* first int32 column of this pass                        */
    uint32_t ncols;           /* valid int32 columns in this pass (<= 4*NV)             */
    int depth;                /* log2 n                                                 */
    const GroupDesc *groups;  /* grouped modes: [key_groups] descriptors (else null)    */
    PhaseParams main;         /* the phase that produces the result (or, in the stand-alone
                                 frontier kernel, the frontier)                          */
    /* single-launch pipeline: the launch first clears its own accumulators and ticket
     * counters and expands the top of every key's tree into the frontier (phase `top`,
     * full seeds), crosses a grid-wide barrier (cooperative launch, every block resident)
     * and then runs `main` from the frontier nodes.                                      */
    int fuse_top;             /* 1: run `top`, barrier, then `main`                      */
    PhaseParams top;
    uint32_t *zero_a;         /* words cleared before the barrier: the result ...        */
    uint64_t zero_a_words;
    uint32_t *zero_b;         /* ... and the main-phase ticket counters                  */
    uint64_t zero_b_words;
    uint32_t *rearm;          /* top-phase tickets, cleared AFTER the barrier for the next launch */
    uint32_t rearm_words;
    uint32_t *grid_bar;       /* monotonic arrival counter of the context               */
    uint32_t grid_bar_target; /* value it reaches when every block of this launch arrived */
    uint32_t top_block_quota; /* tickets one block may draw in the first, balanced round of `top`
                                 (ceil(items / blocks)): the top of the tree is little work, and
                                 first-come-first-served would pile it onto the blocks that start
                                 first; a second, unrestricted round mops up anything left        */
    unsigned long long *timing; /* optional [blocks][8] %globaltimer stamps: start, tables built,
                                 top done, barrier passed, end                                    */
    uint4 *frontier_out;      /* frontier written by `top` (or by the stand-alone kernel) */
    uint32_t nfront;          /* frontier nodes per key (this shard)                    */
    /* wide entries: the first pass also stores every leaf's low word, [key group][leaf
     * position][32 keys], so further column blocks are MAC-only (launch_mac)          */
    uint32_t *leaf_cache;
    uint64_t n_local;         /* leaves in this shard                                   */
    /* expand mode (non-fused): shares[key][index], natural order                      */
    uint32_t *shares;
    uint64_t n;
    /* dynamic shared memory plan (byte offsets from the dynamic smem base)            */
    uint32_t off_cw;          /* uint4 [depth][2 banks][2 bits][32 keys]                */
    uint32_t off_cwlo;        /* uint32 [2][2][32]: low words of the level-0 words      */
    uint32_t off_root;        /* uint4 [32] root seeds                                  */
    uint32_t off_flag;        /* int                                                    */
    uint32_t off_stack_lo;    /* pending-sibling stack, levels [0, stack_split)         */
    uint32_t off_stack_hi;    /* levels [stack_split, s-1)                              */
    uint32_t off_tab;         /* AES tables: 128 KiB whose shared-window address is a
                                 multiple of 64 KiB                                     */
    uint32_t off_tile;        /* MODE_FUSED_TMA: per warp, one work item's rows (64 << s bytes),
                                 then one 8-byte mbarrier per warp at off_tile_bar        */
    uint32_t off_tile_bar;
    /* modes that draw work units: the list, drawn through main.counters[0] (one counter per pass) */
    const WorkUnit *units;
    uint32_t nunits;
    /* modes whose counts are on the device (ModeTraits::counts_on_device): [0] the key groups of `groups`, [1] the
     * work units of `units`, written by the plan kernels (dpf_group_plan.cu).  key_groups and nunits above are then
     * only bounds of those lists */
    const uint32_t *dev_counts;
};

/* Kernel modes: the MODE of dpf_eval_kernel<PRF, NV, MODE>.  Each is a combination of the properties
 * of ModeTraits, and mode_traits below is the one place that says which. */
enum { MODE_FUSED = 0, MODE_EXPAND = 1, MODE_FRONTIER = 2, MODE_GROUPED = 3, MODE_FUSED_TMA = 4,
       MODE_FUSED_ET = 5, MODE_EXPAND_ET = 6, MODE_FUSED_COLSPLIT = 7, MODE_GROUPED_ET = 8,
       MODE_FUSED_XOR = 9, MODE_EXPAND_XOR = 10, MODE_GROUPED_XOR = 11,
       /* the grouped modes with their key-group and work-unit counts on the device (b200dpf_group_eval_device_bins) */
       MODE_GROUPED_DEV = 12, MODE_GROUPED_ET_DEV = 13, MODE_GROUPED_XOR_DEV = 14, MODE_COUNT = 15 };

/* The group a mode's result lives in (ModeTraits::result). */
enum { RESULT_ADD,        /* Z/2^32: out[key][col] = sum of share * row, red.global.add */
       RESULT_XOR };      /* (Z/2)^32: out[key][col] = XOR of the rows whose share bit is set, red.global.xor;
                           * the shares are bits, packed 32 to a word (XOR-shared keys, DESIGN.md section 10) */

/* What a mode's leaves feed (ModeTraits::feeds). */
enum { FEEDS_MAC,         /* the inner product against the table: out[key][col] */
       FEEDS_SHARES,      /* the share vector, shares[key][index] in natural order */
       FEEDS_FRONTIER };  /* whole seeds of the frontier nodes (frontier_out) */
/* How a table row reaches the registers of a FEEDS_MAC mode (ModeTraits::row_load). */
enum { ROWS_BROADCAST,    /* every lane loads the whole row: one broadcast load serves the warp's keys */
       /* the four lanes of a key quad split each row, lane L loading columns 4 (L & 3) .. +3, and the
        * quad's leaf values travel by SHFL instead, so a row costs the shared-memory data pipe one
        * 16-byte load per lane, not four (AES binds that pipe) */
       ROWS_COLSPLIT,
       /* each work item's rows are staged into shared memory by one cp.async.bulk (TMA) when the item
        * is drawn (16-column tables, whole-warp key groups; AES has no shared memory left for them) */
       ROWS_STAGED };

struct ModeTraits {
    int feeds;                /* FEEDS_*                                                          */
    int row_load;             /* ROWS_*                                                           */
    /* log2 table rows per leaf: 2 for early-terminated keys and 7 for XOR-shared ones, whose tree is
     * over leaves while the table, the leaf cache (EvalParams::n_local), the result and the shares
     * (EvalParams::n) are over rows: leaf position p owns rows 4p..4p+3 (128p..128p+127) of the device
     * table, shares[key][4 * leaf + l] */
    int row_shift;
    /* batch PIR: each key group evaluates its own bin, described by EvalParams::groups */
    bool grouped;
    int result;               /* RESULT_*: also the level-0 group, XOR for RESULT_XOR */
    /* the main phase draws work units (EvalParams::units, one per block and draw) instead of walking
     * every key group's tickets: a block touches only the key groups it draws units of */
    bool units;
    /* grouped: the main phase takes its key-group count (units: its work-unit count) from EvalParams::dev_counts, read
     * once per phase, instead of from key_groups (nunits), which is then a bound: the lists were planned on the device */
    bool counts_on_device;
};

__host__ __device__ constexpr ModeTraits mode_traits(int mode)
{
    switch (mode) {                            /* feeds           row_load        row_shift grouped result   units  counts_on_device */
    case MODE_FUSED:          return ModeTraits{FEEDS_MAC,      ROWS_BROADCAST, 0, false, RESULT_ADD, false, false};
    case MODE_EXPAND:         return ModeTraits{FEEDS_SHARES,   ROWS_BROADCAST, 0, false, RESULT_ADD, false, false};
    case MODE_FRONTIER:       return ModeTraits{FEEDS_FRONTIER, ROWS_BROADCAST, 0, false, RESULT_ADD, false, false};
    case MODE_GROUPED:        return ModeTraits{FEEDS_MAC,      ROWS_BROADCAST, 0, true,  RESULT_ADD, false, false};
    case MODE_FUSED_TMA:      return ModeTraits{FEEDS_MAC,      ROWS_STAGED,    0, false, RESULT_ADD, false, false};
    case MODE_FUSED_ET:       return ModeTraits{FEEDS_MAC,      ROWS_BROADCAST, 2, false, RESULT_ADD, false, false};
    case MODE_EXPAND_ET:      return ModeTraits{FEEDS_SHARES,   ROWS_BROADCAST, 2, false, RESULT_ADD, false, false};
    case MODE_FUSED_COLSPLIT: return ModeTraits{FEEDS_MAC,      ROWS_COLSPLIT,  0, false, RESULT_ADD, false, false};
    case MODE_GROUPED_ET:     return ModeTraits{FEEDS_MAC,      ROWS_BROADCAST, 2, true,  RESULT_ADD, false, false};
    case MODE_FUSED_XOR:      return ModeTraits{FEEDS_MAC,      ROWS_COLSPLIT,  7, false, RESULT_XOR, false, false};
    case MODE_EXPAND_XOR:     return ModeTraits{FEEDS_SHARES,   ROWS_BROADCAST, 7, false, RESULT_XOR, false, false};
    case MODE_GROUPED_XOR:    return ModeTraits{FEEDS_MAC,      ROWS_COLSPLIT,  7, true,  RESULT_XOR, true,  false};
    case MODE_GROUPED_DEV:    return ModeTraits{FEEDS_MAC,      ROWS_BROADCAST, 0, true,  RESULT_ADD, false, true};
    case MODE_GROUPED_ET_DEV: return ModeTraits{FEEDS_MAC,      ROWS_BROADCAST, 2, true,  RESULT_ADD, false, true};
    case MODE_GROUPED_XOR_DEV: return ModeTraits{FEEDS_MAC,     ROWS_COLSPLIT,  7, true,  RESULT_XOR, true,  true};
    default:                  return ModeTraits{-1, -1, 0, false, RESULT_ADD, false, false};
    }
}

/* The level-0 group of a mode's keys (dpf_core.cuh GROUP_*) */
__host__ __device__ constexpr int mode_leaf_group(int mode)
{
    return mode_traits(mode).result == RESULT_XOR ? GROUP_XOR128
         : mode_traits(mode).row_shift != 0       ? GROUP_LANES32 : GROUP_ADD128;
}

/* Block shape of the evaluation kernel instantiated for (prf, nv, mode), nv = uint4 (4 int32 columns)
 * of a table row handled per pass: 4, 8 or 16.  The kernel's __launch_bounds__ and the host's grid
 * and shared-memory plan both read it.  AES needs 128 KiB of the SM's shared memory for its tables,
 * so one block per SM; accumulators (4*nv registers) decide how many threads fit the register file.
 * The column-split AES kernel holds 4 row words per leaf instead of 16 and fits 128 registers. */
#ifndef DPF_AES_THREADS
#define DPF_AES_THREADS 384      /* 12 warps: on an H100 1.5 % (n=2^20) and 3 % (n=2^16) faster than 8 (256) */
#endif
struct BlockShape {
    int threads, min_blocks;     /* threads per block, minimum resident blocks per SM */
};
__host__ __device__ constexpr BlockShape eval_block_shape(int prf, int nv, int mode)
{
    if (prf == PRF_AES128)
        return BlockShape{mode_traits(mode).row_load == ROWS_COLSPLIT ? 512 : nv <= 8 ? DPF_AES_THREADS : 256, 1};
    return BlockShape{nv <= 8 ? 256 : 384, nv <= 8 ? 2 : 1};
}

/* Shared-window address of the first dynamic shared memory byte (probed). */
cudaError_t probe_dynamic_smem_base(uint32_t *base, cudaStream_t stream);

/* Upload the AES T-table to this device's constant memory. */
cudaError_t upload_aes_table(const uint32_t *te0_256);

/* One pass of the evaluation kernel of (prf, nv, mode); cudaErrorInvalidValue when that kernel is not
 * instantiated (the table is in dpf_kernels.cu).
 * grid = number of persistent blocks; smem_bytes = dynamic shared memory.  With p.fuse_top the
 * launch is cooperative (every block resident), which the in-kernel grid barrier relies on. */
cudaError_t launch_eval(int prf, int nv, int mode, const EvalParams &p, int grid, size_t smem_bytes,
                        cudaStream_t stream);

/* MAC-only pass over cached leaves: out[key][col_off + c] += sum_pos leaf[kg][pos][key] *
 * table[pos][col_off + c] for the nv*4 columns starting at col_off_v (nv = 4, 8 or 16). */
struct MacParams {
    const uint32_t *leaf_cache;   /* [key_groups][n_local][32] */
    const uint4 *table;
    uint32_t row_stride_v, col_off_v;
    uint32_t *out;
    uint32_t out_stride, col_off, ncols;
    uint32_t col_skip;            /* leading columns of the slice that another pass already produced */
    int nkeys, key_groups;
    uint64_t n_local;
    uint32_t ranges_per_group;    /* position ranges a key group is cut into (one warp each) */
};
cudaError_t launch_mac(int nv, const MacParams &p, int grid, cudaStream_t stream);
/* Same pass (64 columns) with the operands staged into shared memory by cp.async.bulk
 * (TMA) under mbarriers: 8 key groups per block share every staged row slice. */
cudaError_t launch_mac_tma(const MacParams &p, int grid, cudaStream_t stream);

/* Cross-GPU reduction of entry-range partials inside one process: dst[i] += sum_k parts.p[k][i]
 * (mod 2^32).  The kernel runs on the GPU that owns dst and LOADS the other GPUs' partial results
 * through NVLink peer mappings -- no staging copies, no collective library. */
struct PeerParts {
    const uint32_t *p[15];
    int n;
};
cudaError_t launch_sum_partials(uint32_t *dst, const PeerParts &parts, size_t words, int sm_count, cudaStream_t stream);

/* Batched key generation on the device (dpf_keygen.cu): one thread per key pair, ChaCha20-DRBG draws
 * from 44 seed bytes per key, level 0 in `group` (GROUP_*, the kind's), trees of depth + lane_bits bits of
 * alpha.  A flat batch (bins == null) makes `count` keys of one depth, alphas[k] and seeds44[44 k], into
 * [count][131] wire-format slots.  A query batch makes key g of query q at thread k = g * nq + q, from
 * alphas [nq][nbins] and seeds44 [nq][nbins][44], depth bins[g].y, into the wire format [nq][nbins][131]
 * or (compact) the b200dpf_key_pack bytes at uint4 offset q * query_v + bins[g].x, magic in the header. */
struct KeygenParams {
    const int64_t *alphas;
    const uint8_t *seeds44;
    int64_t count;
    int depth, lane_bits;      /* depth: flat batches only */
    const uint2 *bins;         /* query batches: [nbins] (uint4 offset of the key in a compact query, depth) */
    /* query batches: [nbins] the bins' placements.  Key g of query q of a trimmed bin (depth PLACE_IDENTITY) is for
     * row alphas[q][g] mod n (non-negative), at index trimmed_alpha of it; of any other bin for the low bits of alpha */
    const RowPlacement *bin_place;
    uint32_t nq, nbins;
    uint64_t query_v;          /* uint4 per compact query */
    int compact;
    uint32_t magic;            /* compact: the kind's, little-endian */
    const uint32_t *te0;       /* AES Te0, 256 words of global memory */
    uint4 *out_a, *out_b;
};
cudaError_t launch_keygen(int prf, int group, const KeygenParams &p, cudaStream_t stream);

/* The device-planned grouped modes are their parents in every other property, so they take their parents' block
 * shapes: the host plans their grid and shared memory before it knows any count */
static_assert(eval_block_shape(PRF_AES128, 4, MODE_GROUPED_DEV).threads == eval_block_shape(PRF_AES128, 4, MODE_GROUPED).threads &&
              eval_block_shape(PRF_AES128, 4, MODE_GROUPED_ET_DEV).threads == eval_block_shape(PRF_AES128, 4, MODE_GROUPED_ET).threads &&
              eval_block_shape(PRF_AES128, 4, MODE_GROUPED_XOR_DEV).threads == eval_block_shape(PRF_AES128, 4, MODE_GROUPED_XOR).threads &&
              eval_block_shape(PRF_CHACHA20, 4, MODE_GROUPED_XOR_DEV).threads == eval_block_shape(PRF_CHACHA20, 4, MODE_GROUPED_XOR).threads,
              "a device-planned grouped mode has its parent's block shape");

/* Maximum dynamic shared memory the evaluation kernel may be given. */
cudaError_t eval_max_smem(int prf, int nv, int mode, int *bytes);

/* Table creation, one chunk of P's own rows: the rows of P, or of its shard the leaves own_val + k * 2^shift, in natural
 * order.  Own row j = first + q, held at chunk[q][0, cols), goes to device row P.device_row of its natural row
 * ((((j >> lane_bits) << shift) | own_val) << lane_bits) | (j & (2^lane_bits - 1)).  Padded columns [cols, stride) and
 * padding rows are left untouched (pre-zeroed).  The grid-stride helpers take the device's SM count to cap their grids
 * at a few waves. */
cudaError_t launch_fill_table(const int32_t *chunk, uint64_t first, uint64_t count, int32_t *table, const RowPlacement &P,
                              int cols, int stride, int sm_count, cudaStream_t stream);

/* Device-resident grouped evaluation (dpf_group_io.cu), one warp per key, no host synchronisation.
 * order[pos] = (the caller's index of the key at bin-sorted position pos, the depth of its bin).
 *   gather : compact[pos] = the compact form of keys[order[pos].x] (wire format, 131 uint4 each) for a tree
 *            of depth order[pos].y, with `magic` (the kind's, little-endian) in its header, stride_v uint4
 *            apart: the bytes pack_compact writes on the host.
 *   scatter: out[order[pos].x][c] = sorted[pos][c] for c < entry_size (int32 rows). */
cudaError_t launch_group_gather(const void *keys, const uint2 *order, int64_t nkeys, uint32_t magic, uint32_t stride_v,
                                void *compact, cudaStream_t stream);
cudaError_t launch_group_scatter(const int32_t *sorted, const uint2 *order, int64_t nkeys, int entry_size, void *out,
                                 cudaStream_t stream);
/* Queries of one compact key per bin (b200dpf_group_eval_queries_device), nq of them, query_v uint4 each;
 * bins[g] = (uint4 offset of bin g's key in a query, depth of bin g).  compact[g * nq + q] = key g of query q,
 * its header rewritten to (magic, depth, 0, 0), stride_v uint4 apart: the bytes pack_compact writes. */
cudaError_t launch_group_gather_queries(const void *queries, const uint2 *bins, int64_t nkeys, uint32_t nq, uint64_t query_v,
                                        uint32_t magic, uint32_t stride_v, void *compact, cudaStream_t stream);

/* One bin of a grouped context as the device planner sees it, made at create and never rewritten. */
struct GroupBinInfo {
    uint64_t table_off_v;     /* the bin's first row, in uint4 units from the table (GroupDesc::table_off_v) */
    uint32_t rows;            /* rows of its device table, padding included                               */
    int32_t depth;            /* leaf levels of its key tree                                             */
    int32_t room;             /* log2 leaves of the largest work item inside its rows                    */
    uint32_t pad;
};

/* The plan of a grouped evaluation made on the device from a device-resident bin list
 * (b200dpf_group_eval_device_bins, dpf_group_plan.cu).  The host fills what needs no key counts; the kernels
 * compute, from the counts, the lists GroupLaunch::plan makes on the host for the same bins:
 *   histogram : hist[g] = keys of bin g, hist[nbins] = keys whose bin is outside [0, nbins)
 *   sort      : a stable radix sort of (bin, caller's index), out-of-range keys as bin nbins, so they form a tail
 *               no key group covers; order[pos] = (caller's index, bin depth, 0 for the tail)
 *   plan      : one block: s_group by shrink_s, per bin its first sorted key, key group and work unit
 *               (bin_first[g] = (key, group, unit, s)); counts = (key groups, work units, out-of-range keys,
 *               items per unit); *bad = counts[2] when bad is not null
 *   emit      : descs[k] for k < counts[0] in bin order and, for modes that draw work units, units[u] for
 *               u < counts[1] in group-major order */
struct GroupPlanParams {
    const int32_t *bins;      /* [nkeys] the caller's bin ids */
    int64_t nkeys;
    int nbins;
    const GroupBinInfo *bin_info;   /* [nbins] */
    int lane_bits;
    int s_start;              /* s_group before shrink_s: min(subtree_log2 knob or 6, s_max) */
    int shrink;               /* automatic s: shrink from s_start down to s_floor while the launch has fewer items than wanted */
    int s_floor;
    int64_t items_wanted;
    int units;                /* the mode draws work units (ModeTraits::units) */
    int grid, unit_cap;       /* work units: items per unit = clamp(ceil(items / grid), 1, unit_cap) */
    int end_bit;              /* bits of a sort key: bins 0 .. nbins */
    uint32_t *hist;           /* [nbins + 1], cleared by launch_group_plan */
    uint32_t *keys_in, *keys_out, *vals_in, *vals_out;   /* [nkeys] sort buffers */
    void *temp;
    size_t temp_bytes;        /* group_plan_temp_bytes */
    uint4 *bin_first;         /* [nbins] */
    uint2 *order;             /* [nkeys] */
    GroupDesc *descs;         /* [key-group bound] */
    WorkUnit *units_out;      /* [work-unit bound] */
    int64_t descs_cap, units_cap;
    uint32_t *counts;         /* [4] */
    int64_t *bad;             /* or null */
};
/* Bytes of temporary storage the sort of `nkeys` keys below 2^end_bit needs. */
cudaError_t group_plan_temp_bytes(int64_t nkeys, int end_bit, size_t *bytes);
/* Enqueue the histogram, the sort, the plan and the emission on `stream`; no host synchronisation. */
cudaError_t launch_group_plan(const GroupPlanParams &p, int sm_count, cudaStream_t stream);

/* Row update of a live table (b200dpf_update_rows*): device row P.device_row(idx[j]) := rows[j] for j < count, the
 * last occurrence of a device row winning.  P is bin_place[bins[j]] on a grouped context, else `place`; entry j is
 * skipped, never written, when bins[j] is not in [0, nbins) or P does not own idx[j]. */
struct UpdateParams {
    const int64_t *idx;       /* [count] natural rows                                         */
    const int32_t *bins;      /* [count] bin ids, or null                                     */
    const RowPlacement *bin_place;   /* [nbins] the bins' placements                          */
    int nbins;
    RowPlacement place;       /* the context's own placement (bins == null)                   */
    const int32_t *rows;      /* [count][cols] new rows                                       */
    int64_t count;            /* <= 2^31 - 1                                                  */
    uint32_t table_rows;      /* rows of the device table: the skip marker, larger than every device row */
    int32_t *table;           /* [table_rows][stride], 64-byte rows; pad columns are not touched */
    int cols, stride;
};
/* Device scratch of one update: positions and occurrence numbers before and after the sort, then
 * the sort's temporary storage (update_temp_bytes). */
struct UpdateWork {
    uint32_t *pos_in, *pos_out, *ord_in, *ord_out;
    void *temp;
    size_t temp_bytes;
};
/* Bytes of temporary storage the stable sort of `count` positions below 2^end_bit needs. */
cudaError_t update_temp_bytes(int64_t count, int end_bit, size_t *bytes);
/* map -> stable radix sort of (position, occurrence) -> one warp per surviving row; enqueued on
 * `stream`, no host synchronisation. */
cudaError_t launch_update_rows(const UpdateParams &u, const UpdateWork &w, int end_bit, int sm_count, cudaStream_t stream);

/* Batch-code contexts (dpf_batchcode.cu).
 *   scatter: rows [first, first + count) of the table, src holding them [count][cols]: copy c of row r goes to device row
 *            place[bin].first + in-bin row of L.locate(c, r), columns [0, cols) of a stride-int32 row.  One warp per row.
 *   plan   : batchcode_plan_query for each of nq queries, one thread each: wanted [nq][k] -> alphas [nq][nbins], slots
 *            [nq][k]. */
cudaError_t launch_batchcode_scatter(const int32_t *src, uint64_t first, uint64_t count, const BatchCodeLayout &L,
                                     const RowPlacement *place, int32_t *table, int cols, int stride, cudaStream_t stream);
cudaError_t launch_batchcode_plan(const BatchCodeLayout &L, const int64_t *wanted, int64_t nq, int k, int64_t *alphas,
                                  int32_t *slots, cudaStream_t stream);

/* Keyword-PIR contexts (dpf_kwpir.cu); every launch is enqueued on `stream` with no host synchronisation.
 *   check  : radix-sort keys [n] into sorted and set *flags to KWPIR_DUPLICATE and/or KWPIR_RESERVED when two keywords
 *            are equal or one is 2^64 - 1; temp holds kwpir_check_temp_bytes(n) bytes.
 *   round  : round `round` (>= 1) of the placement: the count items of homeless (null: items 0..count-1) bid for slot
 *            choice[i] * m + h_choice[i](keys[i]) (bid words (round << 32) | ~i, atomicMax: the smallest index wins);
 *            each winner takes its slot in owner, and each loser and evicted owner advances its choice and is
 *            appended to next, counted in *next_count (zero before the launch).
 *   scatter: items [first, first + count), values holding their rows [count][L.value_size]: item i's value and tag go
 *            to device row place[choice[i]].first + h_choice[i](keys[i]) of a stride-int32 row.  One warp per item.
 *   plan   : rows3[q][c] = h_c(keywords[q]) for nq queries, one thread each.
 *   find   : bins[j], rows[j] = the table and row whose tag is keywords[j] + 1, or -1, -1; one thread per keyword. */
enum { KWPIR_DUPLICATE = 1, KWPIR_RESERVED = 2 };
cudaError_t kwpir_check_temp_bytes(uint64_t n, size_t *bytes);
cudaError_t launch_kwpir_check(const uint64_t *keys, uint64_t n, uint64_t *sorted, void *temp, size_t temp_bytes, uint32_t *flags,
                               cudaStream_t stream);
cudaError_t launch_kwpir_round(const KeywordLayout &L, const uint64_t *keys, const uint32_t *homeless, uint32_t count,
                               uint32_t round, uint8_t *choice, unsigned long long *bid, int32_t *owner, uint32_t *next,
                               uint32_t *next_count, cudaStream_t stream);
cudaError_t launch_kwpir_scatter(const int32_t *values, uint64_t first, uint64_t count, const uint64_t *keys, const uint8_t *choice,
                                 const KeywordLayout &L, const RowPlacement *place, int32_t *table, int stride, cudaStream_t stream);
cudaError_t launch_kwpir_plan(const KeywordLayout &L, const uint64_t *keywords, int64_t nq, int64_t *rows3, cudaStream_t stream);
cudaError_t launch_kwpir_find(const KeywordLayout &L, const uint64_t *keywords, int64_t count, const RowPlacement *place,
                              const int32_t *table, int stride, int32_t *bins, int64_t *rows, cudaStream_t stream);

}  // namespace b200dpf
