/*
 * dpf_plan.cu -- the launch planner and launcher behind the C ABI: the kernels' shared-memory layouts, the plans
 * of plain and grouped evaluations (EvalPlan, dpf_ctx.h), and launch_plan, which carries a plan out.
 */
#include "dpf_ctx.h"

#include <cmath>
#include <new>

namespace {

int smem_layout_compute(b200dpf_ctx *c, int prf, int nv, int mode, SmemLayout *L)
{
    std::memset(L, 0, sizeof *L);
    const BlockShape shape = eval_block_shape(prf, nv, mode);
    L->threads = shape.threads;
    L->blocks_per_sm = shape.min_blocks;
    L->grid = c->sm_count * L->blocks_per_sm;
    int max_smem = 0;
    CUDA_TRY(eval_max_smem(prf, nv, mode, &max_smem));
    int sm_total = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&sm_total, cudaDevAttrMaxSharedMemoryPerMultiprocessor, c->device));
    /* every resident block also pays the 1 KiB system reservation */
    int budget = std::min(max_smem, sm_total / L->blocks_per_sm - 1024);
    budget &= ~15;
    L->budget = budget;

    L->meta_cw = (uint32_t)c->shape.depth * 4u * 32u * 16u;
    const uint32_t kMetaSmall = 512u + 512u + 16u;
    const uint32_t meta = L->meta_cw + kMetaSmall;
    L->level_bytes = (uint32_t)L->threads * 16u;
    if (prf == B200DPF_PRF_AES128) {
        /* tables: 128 KiB whose shared-window address is 64 KiB aligned */
        const uint32_t tab_abs = (c->smem_base + 65535u) & ~65535u;
        const uint32_t off_tab = tab_abs - c->smem_base;
        const uint32_t a_size = off_tab;                         /* region A: before the tables */
        const uint32_t b_off = off_tab + 131072u;                /* region B: after them        */
        if ((int64_t)budget < (int64_t)b_off) return fail(B200DPF_ECUDA, "shared memory too small for AES tables");
        const uint32_t b_size = (uint32_t)budget - b_off;
        L->off_tab = off_tab;
        uint32_t a_used = 0, b_used = 0;
        if (meta <= a_size) { L->off_meta = 0; L->off_small = L->meta_cw; a_used = meta; }
        else if (meta <= b_size) { L->off_meta = b_off; L->off_small = b_off + L->meta_cw; b_used = meta; }
        else if (L->meta_cw <= a_size && kMetaSmall <= b_size) {
            /* depth 31: the correction words alone fill region A, so the rest goes after the tables */
            L->off_meta = 0; a_used = L->meta_cw;
            L->off_small = b_off; b_used = kMetaSmall;
        }
        else return fail(B200DPF_EINVAL, "depth %d needs more shared memory than available", c->shape.depth);
        a_used = (a_used + 15u) & ~15u;
        b_used = (b_used + 15u) & ~15u;
        L->off_lo = b_off + b_used;
        L->cap_lo = (int)((b_size - b_used) / L->level_bytes);
        L->off_hi = a_used;
        L->cap_hi = (int)((a_size - a_used) / L->level_bytes);
        L->smem_fixed = (size_t)budget;
    } else {
        L->off_meta = 0;
        L->off_small = L->meta_cw;
        L->off_lo = (meta + 15u) & ~15u;
        if ((int64_t)budget < (int64_t)L->off_lo) return fail(B200DPF_EINVAL, "depth %d needs more shared memory than available", c->shape.depth);
        L->cap_lo = (int)(((uint32_t)budget - L->off_lo) / L->level_bytes);
        L->off_hi = L->off_lo;
        L->cap_hi = 0;
        L->smem_fixed = 0;
    }
    L->s_max = 1 + L->cap_lo + L->cap_hi;
    return B200DPF_OK;
}

/* Dynamic shared memory of a launch on layout L whose deepest pending-sibling stack is s levels */
size_t smem_bytes(const SmemLayout &L, int s)
{
    return L.smem_fixed ? L.smem_fixed : (size_t)L.off_lo + (size_t)(s > 1 ? s - 1 : 0) * L.level_bytes;
}

void fill_phase(const SmemLayout &L, int s, PhaseParams *ph)
{
    std::memset(ph, 0, sizeof *ph);
    ph->s = s;
    ph->stack_split = std::min(L.cap_lo, std::max(s - 1, 0));
}

/* Work-item size: from s down to s_floor, the first s at which the launch has at least `wanted` items */
template <class Items> int shrink_s(int s, int s_floor, int64_t wanted, Items items)
{
    while (s > s_floor && items(s) < wanted) s--;
    return s;
}

/* The fields of EvalParams that every launch of job J on layout L shares; the others are zero. */
void fill_common(const b200dpf_ctx *c, const SmemLayout &L, const EvalJob &J, const EvalPlan &P, EvalParams *p)
{
    std::memset(p, 0, sizeof *p);
    p->keys = reinterpret_cast<const uint4 *>(J.keys);
    p->key_stride_v = J.kl.stride_v; p->key_root_v = J.kl.root_v; p->key_compact = J.kl.compact;
    p->depth = c->shape.depth;
    p->nkeys = (int)J.nkeys; p->kpw_log2 = P.kpw_log2; p->key_groups = (int)P.key_groups;
    p->groups = J.groups; p->units = J.units; p->nunits = J.nunits; p->dev_counts = J.counts;
    p->table = reinterpret_cast<const uint4 *>(c->d_table.ptr);
    p->row_stride_v = (uint32_t)c->entry_pad / 4u;
    p->out_stride = (uint32_t)c->entry_size;
    p->n = (uint64_t)c->shape.n;
    p->off_cw = L.off_meta;
    p->off_cwlo = L.off_small;
    p->off_root = p->off_cwlo + 512u;
    p->off_flag = p->off_root + 512u;
    p->off_stack_lo = L.off_lo;
    p->off_stack_hi = L.off_hi;
    p->off_tab = L.off_tab;
}

/* The plan of job J on a plain context. */
int plan_eval(b200dpf_ctx *c, const EvalJob &J, EvalPlan *out)
{
    const b200dpf_ctx::Knobs &K = c->knobs;
    const KindOps &ops = kKindOps[c->kind];
    const int prf = J.prf;
    const int64_t nkeys = J.nkeys;
    const bool fused = J.mode_main == MODE_FUSED;
    EvalPlan &P = *out = EvalPlan{};
    int &kpw_log2 = P.kpw_log2, &s = P.s, &f_rel = P.f_rel, &s_top = P.s_top;   /* the names the arithmetic below uses */
    int64_t &key_groups = P.key_groups;
    SmemLayout &L = P.L;
    P.leaf_cache = J.leaf_cache;
    /* Entries wider than 32 columns: the tree is expanded ONCE by the best-shaped kernel (16
     * columns, NV = 4), which also caches each leaf's low word; every other column is produced by
     * MAC-only passes over that cache.  Without the cache (disabled or lane-split batches) wide
     * entries use one tree expansion per 64 columns. */
    P.nv = (!fused || c->entry_pad <= 16 || P.leaf_cache) ? 4 : std::min(ops.max_nv, c->entry_pad <= 32 ? 8 : 16);
    P.passes = fused ? (P.leaf_cache ? 1 : c->entry_pad / (4 * P.nv)) : 1;
    /* optional variant: the rows of each work item staged into shared memory by cp.async.bulk */
    P.tma_rows = K.tma_rows != 0 && K.one_launch != 0 && c->coop_ok != 0 && fused && c->entry_pad == 16 &&
                 prf != B200DPF_PRF_AES128 && nkeys >= 17 && ops.tma_rows;
    const int mode_plain = fused ? ops.mode_fused : ops.mode_expand;
    P.mode = P.tma_rows ? MODE_FUSED_TMA : mode_plain;
    /* keys per warp: a full warp of keys when the batch allows; for small batches the
     * spare lanes take adjacent subtrees of the same keys (single-query latency mode) */
    kpw_log2 = 5;
    if (K.lane_split != 0)
        while (kpw_log2 > 0 && ((int64_t)1 << (kpw_log2 - 1)) >= nkeys) kpw_log2--;
    if (fused) kpw_log2 = std::max(kpw_log2, ops.min_kpw_log2);
    key_groups = (nkeys + ((int64_t)1 << kpw_log2) - 1) >> kpw_log2;
    /* AES binds the shared-memory data pipe, and a broadcast row load is charged for every lane's copy
     * of the row: with at least 4 keys per warp, each lane of a key quad loads a quarter of the row and
     * the quad trades leaf values by SHFL instead (DESIGN.md section 3).  Decided before the layout: the
     * kernel runs more threads, so its stack holds fewer levels (s_max).  kpw_log2 only grows below. */
    if (P.mode == MODE_FUSED && prf == B200DPF_PRF_AES128 && P.nv == 4 && kpw_log2 >= 2)
        P.mode = MODE_FUSED_COLSPLIT;
    int rc = smem_layout(c, prf, P.nv, P.mode, &L);
    if (rc) return rc;
    const int64_t warps = (int64_t)L.grid * (L.threads / 32);

    /* ---- work-item size s and the frontier depth --------------------------------
     * Without a frontier every item re-walks depth-s levels from the root, so items
     * must be big; with one the walk is (almost) free and small items balance the
     * tail. */
    const bool want_frontier = K.frontier != 0;
    if (K.subtree_log2 > 0) {
        s = std::min(K.subtree_log2, std::min(c->depth_local(), L.s_max));
    } else {
        /* B=512 E=16, frontier on, 1x H100 SXM 80 GB at a 400 W power limit, DPFs/s (run-to-run
         * spread about 3 %); the automatic choice is within the spread of the best fixed s:
         *   AES n=2^20: auto 19.47k; s=4 19.39k, 5 19.77k, 6 19.56k, 7 20.01k, 8 19.56k
         *   AES n=2^16: auto 319.3k; s=4 317.5k, 5 318.1k, 6 318.1k, 7 300.5k
         *   ChaCha n=2^20: auto 19.18k; s=5 18.94k, 6 19.13k, 7 19.19k */
        const int s_cap = want_frontier ? 7 : ((prf == B200DPF_PRF_AES128) ? 8 : 10);
        /* XOR-shared keys: a leaf is 128 rows of work, so a few items per warp balance the tail and the
         * smallest items keep every warp busy at small n.  AES, E=16, B=512, H100 80GB HBM3 at a 700 W
         * power limit, SM clock 1980 MHz, ms per batch (DESIGN.md section 10):
         *   n=2^16: auto 0.107; s=1 0.103, 2 0.148, 3 0.196, 4 0.262, 5 0.490
         *   n=2^20: auto 0.971; s=1 0.989, 2 0.980, 3 0.971, 4 0.975, 5 0.975, 6 0.973 */
        const int s_floor = ops.leaf_items ? 1 : want_frontier ? 3 : 5;
        const int64_t items_per_warp = ops.leaf_items ? ops.leaf_items : want_frontier ? 24 : 6;
        s = shrink_s(std::min(c->depth_local(), std::min(L.s_max, s_cap)), s_floor, items_per_warp * warps, [&](int t) {
            return ((c->rows_local() >> (t + c->lane_bits())) * key_groups) >> (5 - kpw_log2);
        });
    }
    if (s < 1) s = 1;
    if (P.tma_rows) {
        /* one tile of 2^s 64-byte rows per warp, after the sibling stack */
        const int warps_blk = L.threads / 32;
        if (K.subtree_log2 <= 0) s = std::min(s, 6);
        P.tile_bytes = (size_t)warps_blk * ((size_t)64 << s) + 8u * (size_t)warps_blk + 16u;
        if ((size_t)L.off_lo + (size_t)(std::max(s, 7) - 1) * L.level_bytes + P.tile_bytes > (size_t)L.budget) {
            P.tma_rows = false;             /* does not fit beside correction words and stack: broadcast loads */
            P.mode = mode_plain;
            P.tile_bytes = 0;
            rc = smem_layout(c, prf, P.nv, P.mode, &L);
            if (rc) return rc;
        }
    }
    if (c->trimmed) {
        /* a ticket (2^(s + spw_log2) leaves) must not reach past the padded rows: smaller items first (down to
         * one leaf pair), then fewer subtrees per warp.  Lanes of a key quad trade leaf values by SHFL, so every
         * lane of an issued ticket runs; the padding is what keeps its rows inside the table. */
        const int room = c->shape.room;
        s = std::max(1, std::min(s, room - (5 - kpw_log2)));
        if (5 - kpw_log2 > room - s) {
            kpw_log2 = 5 - (room - s);
            key_groups = (nkeys + ((int64_t)1 << kpw_log2) - 1) >> kpw_log2;
        }
    }
    const int rel = c->depth_local() - s;           /* tree levels between the shard root and the items */
    if (5 - kpw_log2 > rel) {                     /* not enough subtrees to split a warp that far */
        kpw_log2 = 5 - rel;
        key_groups = (nkeys + ((int64_t)1 << kpw_log2) - 1) >> kpw_log2;
    }
    const int spw_log2 = 5 - kpw_log2;
    if (P.leaf_cache && kpw_log2 != 5) return fail(B200DPF_ESTATE, "internal: leaf cache planned for a lane-split batch");

    if (want_frontier && rel >= 2) {
        const int64_t cap_bytes = (int64_t)K.frontier_mb << 20;
        f_rel = rel;
        while (f_rel > 0 && ((key_groups * (16 << kpw_log2)) << f_rel) > cap_bytes) f_rel--;
        if (f_rel < 2 || f_rel < spw_log2 + 1) f_rel = 0;
    }

    P.one_launch = K.one_launch != 0 && c->coop_ok != 0;
    P.pass_counters = (size_t)key_groups;
    P.top_counters = std::max<size_t>((size_t)key_groups, 64);
    if (f_rel > 0) P.frontier_bytes = ((size_t)key_groups * (16 << kpw_log2)) << f_rel;

    /* ---- the tree-top phase (frontier build) ---- */
    P.LF = L;
    if (f_rel > 0) {
        if (!P.one_launch && (rc = smem_layout(c, prf, 4, MODE_FRONTIER, &P.LF))) return rc;
        const SmemLayout &LF = P.LF;
        s_top = std::max(1, std::min(f_rel - spw_log2, std::min(5, LF.s_max)));
        if (K.top_log2 > 0) {
            s_top = std::max(1, std::min(K.top_log2, std::min(f_rel - spw_log2, LF.s_max)));
        } else if (P.one_launch && K.balance_top) {
            /* Size of a tree-top item.  The blocks that start at a key group share its 2^(f_rel - s_top)
             * items; an item is (walk to its subtree root) + 2^s_top - 1 node pairs, all sequential.
             * Estimate the phase as rounds x steps x step time, where a step costs the larger of the
             * warps sharing the SM's binding pipe and the latency of one dependent expansion, and take
             * the best size: few long items when blocks are plentiful (one round, few busy warps),
             * more short ones when every warp can be given one.  (AES n=2^20 on 8 shards: s_top 6
             * instead of 5 halves the phase; n=2^14, 16 key groups: 5 stays best.) */
            const int nw = L.threads / 32;
            const double blocks_per_group = std::max(1.0, (double)L.grid / (double)key_groups);
            double best = 1e300;
            for (int cand = 1; cand <= std::min(f_rel - spw_log2, std::min(7, LF.s_max)); cand++) {
                const double tickets = (double)((int64_t)1 << (f_rel - cand)) / (double)(1 << spw_log2) *
                                       std::max(1.0, (double)key_groups / (double)L.grid);
                const double quota = std::ceil(tickets / blocks_per_group);
                const double steps = 0.55 * (c->shard_bits + f_rel - cand) + (double)((1 << cand) - 1);
                const double full_rounds = std::floor(quota / nw), rest = quota - full_rounds * nw;
                const double busy = 330.0, latency = 1500.0;        /* per node pair: pipe slots, dependent-chain latency */
                double t = full_rounds * steps * std::max(nw * busy, latency);
                if (rest > 0) t += steps * std::max(rest * busy, latency);
                if (t < best) {
                    best = t;
                    s_top = cand;
                }
            }
        }
        fill_phase(LF, s_top, &P.top);
        P.top.nsub = (uint32_t)1 << (f_rel - s_top);
        P.top.sub_first = (uint32_t)c->shard_rank << (f_rel - s_top);
        P.top.walk_first_level = c->shape.depth - 1;
        P.top.walk_steps = c->shard_bits + f_rel - s_top;
        P.top.level_base = c->depth_local() - f_rel;
        P.smem_top = smem_bytes(LF, s_top);
        P.nfront = (uint32_t)1 << f_rel;
    }

    /* ---- the main phase ---- */
    P.smem = smem_bytes(L, std::max(s, s_top));
    if (P.tma_rows) {
        P.off_tile = (uint32_t)((P.smem + 15) & ~(size_t)15);
        P.off_tile_bar = P.off_tile + (uint32_t)((size_t)(L.threads / 32) * ((size_t)64 << s));
        P.smem = (size_t)P.off_tile + P.tile_bytes;
    }
    fill_phase(L, s, &P.main);
    P.main.nsub = (uint32_t)(c->rows_local() >> (s + c->lane_bits()));   /* 2^rel, or the items over a trimmed table's rows */
    P.main.sub_first = (uint32_t)c->shard_rank << rel;
    if (f_rel > 0) {
        P.main.front_shift = rel - f_rel;
        P.main.walk_first_level = c->depth_local() - f_rel - 1;
        P.main.walk_steps = rel - f_rel;
    } else {
        P.main.walk_first_level = c->shape.depth - 1;
        P.main.walk_steps = c->shape.depth - s;
    }
    if (P.one_launch) {
        const uint64_t items = (uint64_t)key_groups * (uint64_t)(P.top.nsub >> spw_log2);
        P.top_block_quota = K.balance_top ? (uint32_t)std::max<uint64_t>(1, (items + (uint64_t)L.grid - 1) / (uint64_t)L.grid)
                                          : 0x7fffffffu;
        P.timing = K.timing != 0;
    }

    /* ---- wide entries: the leaf-caching pass, then the MAC-only passes ---- */
    if (P.leaf_cache) {
        P.mode = ops.mode_fused;                   /* the kind's fused kernel, on the layout planned above */
        P.leaf_cache_bytes = (size_t)key_groups * 32u * (size_t)c->rows_local() * sizeof(uint32_t);
        P.mac_tma = K.mac_tma != 0;
        /* register-staged variant: 8 warps per block */
        const int64_t mac_warps = (int64_t)c->sm_count * 2 * 8;
        const int64_t ranges = std::max<int64_t>(1, (2 * mac_warps + key_groups - 1) / key_groups);
        /* TMA variant: one block per SM; a block takes 8 key groups x one position range */
        const int64_t kg_blocks = (key_groups + 7) / 8;
        const int64_t tr = std::max<int64_t>(1, (2 * (int64_t)c->sm_count + kg_blocks - 1) / kg_blocks);
        P.mac_grid = P.mac_tma ? c->sm_count : c->sm_count * 2;
        P.mac_ranges = (uint32_t)(P.mac_tma ? std::min<int64_t>(tr, std::max<int64_t>(1, c->rows_local() / 256))
                                            : std::min<int64_t>(ranges, std::max<int64_t>(1, c->rows_local() / 64)));
    }
    return B200DPF_OK;
}

/* The part of a grouped plan that needs no key counts: the mode, the passes, the shared-memory layout and the grid
 * (which depend on the kernel alone, not on s), and s_group before shrink_s.  Automatic s (`shrink`) shrinks it from
 * there down to *s_floor while the launch has fewer than *items_wanted work items. */
int plan_group_base(b200dpf_ctx *c, int prf, int mode, EvalPlan *out, bool *shrink, int *s_floor, int64_t *items_wanted)
{
    const KindOps &ops = kKindOps[c->kind];
    EvalPlan &P = *out = EvalPlan{};
    const SmemLayout &L = P.L;
    P.grouped = P.one_launch = true;
    P.mode = mode;
    P.nv = 4; P.passes = c->entry_pad / 16;     /* 16 columns per pass */
    P.kpw_log2 = 5;
    int rc = smem_layout(c, prf, P.nv, P.mode, &P.L);
    if (rc) return rc;
    const int64_t warps = (int64_t)L.grid * (L.threads / 32);
    P.s_group = std::min(c->knobs.subtree_log2 > 0 ? c->knobs.subtree_log2 : 6, L.s_max);
    *shrink = c->knobs.subtree_log2 <= 0;
    *s_floor = ops.leaf_items ? 1 : 3;
    *items_wanted = (ops.leaf_items ? ops.leaf_items : 2) * warps;
    return B200DPF_OK;
}

}  // namespace

namespace b200dpf::capi {

/* Dynamic shared memory layout of the kernel instantiated for (prf, nv, mode); the CUDA
 * attribute queries behind it are made once per context. */
int smem_layout(b200dpf_ctx *c, int prf, int nv, int mode, SmemLayout *L)
{
    const int ni = nv == 4 ? 0 : (nv == 8 ? 1 : 2);
    if (!c->layouts) c->layouts.reset(new (std::nothrow) SmemLayoutCache());
    if (c->layouts && c->layouts->valid[prf][ni][mode]) {
        *L = c->layouts->entry[prf][ni][mode];
        return B200DPF_OK;
    }
    const int rc = smem_layout_compute(c, prf, nv, mode, L);
    if (rc == B200DPF_OK && c->layouts) {
        c->layouts->entry[prf][ni][mode] = *L;
        c->layouts->valid[prf][ni][mode] = true;
    }
    return rc;
}

/* The plan of one evaluation on a grouped context, whose bin-sorted keys of bin g are at positions
 * count[g] .. count[g + 1].  Key groups and their work-item size: big items amortise the root-to-subtree
 * walk every item pays (there is no frontier: bins are small), small items keep every warp busy.  Leaves
 * of many rows (KindOps::leaf_items) take items down to s = 1, as on a plain context.  One cooperative
 * launch per 16 columns; the first one clears the result and every pass's tickets. */
int plan_group_eval(b200dpf_ctx *c, int prf, const std::vector<int64_t> &count, EvalPlan *out)
{
    const GroupBins *B = c->bins.get();
    const int nbins = (int)B->shape.size();
    EvalPlan &P = *out;
    const SmemLayout &L = P.L;
    bool shrink = false;
    int s_floor = 0;
    int64_t items_wanted = 0;
    int rc = plan_group_base(c, prf, kKindOps[c->kind].mode_grouped, out, &shrink, &s_floor, &items_wanted);
    if (rc) return rc;
    auto groups_of = [&](int g) { return (count[(size_t)g + 1] - count[(size_t)g] + 31) / 32; };
    for (int g = 0; g < nbins; g++) P.key_groups += groups_of(g);
    if (shrink) {
        P.s_group = shrink_s(P.s_group, s_floor, items_wanted, [&](int t) {
            int64_t items = 0;
            for (int g = 0; g < nbins; g++)
                items += groups_of(g) * (B->shape[(size_t)g].rows >> (std::min(B->shape[(size_t)g].room, t) + c->lane_bits()));
            return items;
        });
    }
    P.s = 1;
    for (int g = 0; g < nbins; g++)
        if (count[(size_t)g + 1] > count[(size_t)g]) P.s = std::max(P.s, group_s(P, *B, g));
    /* per pass: one ticket counter per key group, or the one unit counter */
    P.pass_counters = mode_traits(P.mode).units ? 1u : (size_t)P.key_groups;
    P.smem = smem_bytes(L, P.s);
    fill_phase(L, P.s, &P.main);
    return B200DPF_OK;
}

/* The host half of the plan of b200dpf_group_eval_device_bins for nkeys keys: plan_group_base, bounds of the lists
 * the device half writes, and their buffers.  The rest (the counts, s_group, every group's s, the lists) is
 * computed on the device from the bins by launch_group_plan. */
int plan_group_device(b200dpf_ctx *c, int prf, int64_t nkeys, DevicePlanned *D)
{
    GroupBins *B = c->bins.get();
    const int nbins = (int)B->shape.size();
    EvalPlan &P = D->P;
    const SmemLayout &L = P.L;
    D->valid = false;
    bool shrink = false;
    int s_floor = 0;
    int64_t items_wanted = 0;
    int rc = plan_group_base(c, prf, kKindOps[c->kind].mode_grouped_dev, &P, &shrink, &s_floor, &items_wanted);
    if (rc) return rc;
    /* every key group but the last of its bin holds 32 keys: at most nkeys / 32 full groups, and one partial group
     * per bin that has keys */
    P.key_groups = nkeys / 32 + std::min<int64_t>(nbins, nkeys);
    /* shared memory for the largest s a group can be given (group_s <= max(1, s_group)); a group's own s only picks
     * its items.  L.grid and the block shape come from the kernel alone, so they do not depend on s. */
    P.s = std::max(1, P.s_group);
    P.pass_counters = mode_traits(P.mode).units ? 1u : (size_t)P.key_groups;
    P.smem = smem_bytes(L, P.s);
    fill_phase(L, P.s, &P.main);
    /* Work units (GroupLaunch::plan): a key group of nsub items is cut into ceil(nsub / per_unit) units, per_unit =
     * clamp(ceil(items / grid), 1, W) with W warps per block and `items` the sum of every group's nsub.  So units
     * <= key groups + items / per_unit.  While per_unit < W, per_unit >= items / grid and items / per_unit <= grid;
     * at per_unit = W, items / W <= key groups * nsub_max / W, nsub_max being the most items a bin's group can
     * have (at s = 1). */
    const bool units = mode_traits(P.mode).units;
    const int unit_cap = L.threads / 32;
    D->units_bound = 0;
    if (units) {
        int64_t nsub_max = 1;
        for (const TableShape &t : B->shape) nsub_max = std::max<int64_t>(nsub_max, t.rows >> (1 + c->lane_bits()));
        D->units_bound = P.key_groups + std::max<int64_t>(L.grid, (P.key_groups * nsub_max + unit_cap - 1) / unit_cap);
    }
    GroupPlanParams &g = D->gp;
    g = GroupPlanParams{};
    g.nkeys = nkeys;
    g.nbins = nbins;
    g.bin_info = B->d_bin_info.ptr;
    g.lane_bits = c->lane_bits();
    g.s_start = P.s_group;
    g.shrink = shrink ? 1 : 0;
    g.s_floor = s_floor;
    g.items_wanted = items_wanted;
    g.units = units ? 1 : 0;
    g.grid = L.grid;
    g.unit_cap = unit_cap;
    g.end_bit = ilog2((int64_t)nbins + 1);     /* sort keys 0 .. nbins, nbins for a key outside every bin */
    CUDA_TRY(group_plan_temp_bytes(nkeys, g.end_bit, &g.temp_bytes));
    g.descs_cap = P.key_groups;
    g.units_cap = D->units_bound;
    rc = D->d_hist.reserve(((size_t)nbins + 1) * sizeof(uint32_t));
    if (!rc) rc = D->d_counts.reserve(4 * sizeof(uint32_t));
    if (!rc) rc = D->d_bin_first.reserve((size_t)nbins * sizeof(uint4));
    if (!rc) rc = D->d_sort.reserve(4 * (size_t)nkeys * sizeof(uint32_t));
    if (!rc) rc = D->d_temp.reserve(std::max<size_t>(g.temp_bytes, 1));
    if (!rc) rc = D->d_order.reserve((size_t)nkeys * sizeof(uint2));
    if (!rc) rc = D->d_descs.reserve((size_t)P.key_groups * sizeof(GroupDesc));
    if (!rc && units) rc = D->d_units.reserve((size_t)D->units_bound * sizeof(WorkUnit));
    if (rc) return rc;
    g.hist = D->d_hist.ptr;
    g.keys_in = D->d_sort.ptr;
    g.keys_out = g.keys_in + nkeys;
    g.vals_in = g.keys_out + nkeys;
    g.vals_out = g.vals_in + nkeys;
    g.temp = D->d_temp.ptr;
    g.bin_first = D->d_bin_first.ptr;
    g.order = D->d_order.ptr;
    g.descs = D->d_descs.ptr;
    g.units_out = D->d_units.ptr;
    g.counts = D->d_counts.ptr;
    D->nkeys = nkeys;
    D->prf = prf;
    D->valid = true;
    return B200DPF_OK;
}

/* Carry out plan P of job J: reserve what it asks for, order it after the context's last operation, clear,
 * launch and make that the context's last operation.  A device that cannot keep the whole persistent grid
 * resident (a partitioned GPU, say) refuses the first cooperative launch before anything of the evaluation
 * ran: a plain context then falls back, for its life, to separate launches, planned again. */
int launch_plan(b200dpf_ctx *c, const EvalJob &J, const EvalPlan &P)
{
    const bool fused = J.mode_main == MODE_FUSED;
    const size_t n_counters = (size_t)P.passes * P.pass_counters;
    bool grown = false;
    int rc = c->d_counters.reserve(n_counters * sizeof(uint32_t));
    if (!rc && P.top_counters) rc = c->d_top_counters.reserve(P.top_counters * sizeof(uint32_t), &grown);
    if (grown) c->coop_state_dirty = true;
    if (!rc && P.frontier_bytes) rc = c->d_frontier.reserve(P.frontier_bytes);
    if (!rc) rc = wait_last(c, J.stream);
    if (rc) return rc;

    if (!P.one_launch || c->coop_state_dirty) {
        if (P.top_counters) CUDA_TRY(cudaMemsetAsync(c->d_top_counters.ptr, 0, c->d_top_counters.cap, J.stream));
        CUDA_TRY(cudaMemsetAsync(c->d_gridbar.ptr, 0, sizeof(uint32_t), J.stream));
        c->bar_epoch = 0;
        c->coop_state_dirty = false;
    }
    if (!P.one_launch) {
        CUDA_TRY(cudaMemsetAsync(c->d_counters.ptr, 0, n_counters * sizeof(uint32_t), J.stream));
        if (fused && J.clear_out)
            CUDA_TRY(cudaMemsetAsync(J.out, 0, (size_t)J.nkeys * c->entry_size * sizeof(int32_t), J.stream));
        c->coop_state_dirty = true;     /* the stand-alone frontier kernel leaves its tickets used */
    }
    if (P.timing) rc = c->d_timing.reserve((size_t)P.L.grid * 8 * sizeof(unsigned long long));
    if (!rc && P.leaf_cache_bytes) rc = c->d_leaf_cache.reserve(P.leaf_cache_bytes);
    if (rc) return rc;
    if (P.timing) CUDA_TRY(cudaMemsetAsync(c->d_timing.ptr, 0, c->d_timing.cap, J.stream));
    c->last_launches = 0;
    if (J.timed) CUDA_TRY(cudaEventRecord(c->ev_t0, J.stream));

    EvalParams p;
    PhaseParams top = P.top;
    if (P.f_rel > 0) top.counters = c->d_top_counters.ptr;
    uint4 *const frontier = reinterpret_cast<uint4 *>(c->d_frontier.ptr);
    if (P.f_rel > 0 && !P.one_launch) {           /* the stand-alone frontier kernel */
        fill_common(c, P.LF, J, P, &p);
        p.main = top; p.nfront = P.nfront; p.frontier_out = frontier;
        CUDA_TRY(launch_eval(J.prf, 4, MODE_FRONTIER, p, P.LF.grid, P.smem_top, J.stream));
        c->last_launches++;
    }

    fill_common(c, P.L, J, P, &p);
    p.main = P.main;
    p.main.counters = c->d_counters.ptr;
    if (P.f_rel > 0) p.main.frontier_in = frontier;
    p.nfront = P.nfront;
    p.off_tile = P.off_tile; p.off_tile_bar = P.off_tile_bar;
    if (P.one_launch) {
        p.fuse_top = 1;
        if (fused && J.clear_out) { p.zero_a = reinterpret_cast<uint32_t *>(J.out); p.zero_a_words = (uint64_t)J.nkeys * c->entry_size; }
        p.zero_b = c->d_counters.ptr; p.zero_b_words = n_counters;
        if (!P.grouped) {
            p.top = top;                  /* nsub == 0: no frontier, the top phase only clears */
            p.frontier_out = frontier;
            p.rearm = c->d_top_counters.ptr; p.rearm_words = (uint32_t)P.key_groups;
            p.top_block_quota = P.top_block_quota;
        }
        if (P.timing) p.timing = c->d_timing.ptr;
        p.grid_bar = c->d_gridbar.ptr;
        c->bar_epoch += (uint32_t)P.L.grid;
        p.grid_bar_target = c->bar_epoch;
    }

    bool coop_refused = false;
    auto launch_main = [&]() -> int {
        const cudaError_t e = launch_eval(J.prf, P.nv, P.mode, p, P.L.grid, P.smem, J.stream);
        if (e != cudaSuccess) {
            c->coop_state_dirty = true;
            coop_refused = e == cudaErrorCooperativeLaunchTooLarge && p.fuse_top && !P.grouped;
            return fail(B200DPF_ECUDA, "%s: %s", P.grouped ? "grouped evaluation launch" : "evaluation kernel launch",
                        cudaGetErrorString(e));
        }
        c->last_launches++;
        p.fuse_top = 0;                   /* later passes of this evaluation reuse the frontier */
        return B200DPF_OK;
    };
    if (J.mode_main == MODE_EXPAND) {
        p.shares = reinterpret_cast<uint32_t *>(J.out);
        rc = launch_main();
    } else {
        p.out = reinterpret_cast<uint32_t *>(J.out);
        if (P.leaf_cache) { p.leaf_cache = c->d_leaf_cache.ptr; p.n_local = (uint64_t)c->rows_local(); }
        for (int pass = 0; pass < P.passes && rc == B200DPF_OK; pass++) {
            p.col_off_v = (uint32_t)(pass * P.nv);
            p.col_off = (uint32_t)(pass * 4 * P.nv);
            p.ncols = (uint32_t)std::max(0, std::min(4 * P.nv, c->entry_size - pass * 4 * P.nv));
            if (p.ncols == 0) break;
            p.main.counters = c->d_counters.ptr + (size_t)pass * P.pass_counters;
            rc = launch_main();
        }
    }
    if (coop_refused) {
        cudaGetLastError();
        c->coop_ok = 0;
        EvalPlan Q;
        return (rc = plan_eval(c, J, &Q)) ? rc : launch_plan(c, J, Q);
    }
    if (rc) return rc;

    if (P.leaf_cache) {
        MacParams m;
        std::memset(&m, 0, sizeof m);
        m.leaf_cache = p.leaf_cache; m.table = p.table; m.row_stride_v = p.row_stride_v;
        m.out = p.out; m.out_stride = p.out_stride;
        m.nkeys = (int)J.nkeys; m.key_groups = (int)P.key_groups; m.n_local = (uint64_t)c->rows_local();
        m.ranges_per_group = P.mac_ranges;
        for (int blk = 0; blk * 64 < c->entry_size; blk++) {       /* 64-column slices of the rows */
            m.col_off_v = (uint32_t)(blk * 16); m.col_off = (uint32_t)(blk * 64);
            m.ncols = (uint32_t)std::min(64, c->entry_size - blk * 64);
            m.col_skip = blk == 0 ? 16u : 0u;                      /* columns 0..15 came from the fused pass */
            if (m.ncols <= m.col_skip) continue;
            if (P.mac_tma) CUDA_TRY(launch_mac_tma(m, P.mac_grid, J.stream));
            else CUDA_TRY(launch_mac(16, m, P.mac_grid, J.stream));
            c->last_launches++;
        }
    }
    if (J.timed) { CUDA_TRY(cudaEventRecord(c->ev_t1, J.stream)); c->timed = true; }
    return mark_last(c, J.stream);
}

/*
 * One evaluation on a plain context.  Wide entries whose leaf cache (nkeys x rows_local x 4 bytes) would
 * exceed the cap are evaluated in batch chunks that fit -- the cache is what makes columns beyond the
 * first 16 cost a MAC pass instead of a tree expansion, so shrinking the chunk beats dropping the cache.
 */
int run_pipeline(b200dpf_ctx *c, const void *keys_dev, const KeyLayout &kl, int64_t nkeys, int prf, int mode_main,
                 void *out_dev, cudaStream_t stream, bool clear_out)
{
    const b200dpf_ctx::Knobs &K = c->knobs;
    const bool wide = mode_main == MODE_FUSED && c->entry_pad > 32 && nkeys >= 17 && K.leaf_cache != 0 && kKindOps[c->kind].leaf_cache;
    const size_t per_group = 32u * (size_t)c->rows_local() * sizeof(uint32_t);
    const size_t cap = (size_t)std::max(K.leaf_cache_mb, 1) << 20;
    /* not a cached evaluation, or one key group alone overflows the cap (re-expand per 64 columns): one chunk */
    const bool cached = wide && per_group <= cap;
    const int64_t chunk = cached ? (int64_t)std::max<size_t>(1, cap / per_group) * 32 : nkeys;
    EvalJob J{keys_dev, kl, nkeys, prf, mode_main, out_dev, stream, clear_out};
    int rc = B200DPF_OK, launches = 0;
    for (int64_t k0 = 0; k0 < nkeys && rc == B200DPF_OK; k0 += chunk) {
        J.nkeys = std::min(chunk, nkeys - k0);
        J.keys = reinterpret_cast<const char *>(keys_dev) + (size_t)k0 * kl.stride_v * 16u;
        J.out = reinterpret_cast<char *>(out_dev) + (size_t)k0 * c->entry_size * sizeof(int32_t);
        /* a ragged tail below 17 keys would be lane-split, which the cache layout excludes */
        J.leaf_cache = cached && J.nkeys >= 17;
        EvalPlan P;
        rc = plan_eval(c, J, &P);
        if (!rc) rc = launch_plan(c, J, P);
        launches += c->last_launches;
    }
    c->last_launches = launches;
    return rc;
}

}  // namespace b200dpf::capi
