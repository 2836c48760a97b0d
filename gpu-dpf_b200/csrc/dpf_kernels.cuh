/*
 * dpf_kernels.cuh -- launch interface between the C-ABI layer (dpf_capi.cu)
 * and the sm_90a kernels (dpf_kernels.cu).  Plain structs, no torch.
 */
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace b200dpf {

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
    uint32_t nsub;            /* number of 2^s-subtrees in this shard                   */
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
    int32_t depth;            /* log2 of the bin's table size (MODE_GROUPED_ET: of its leaves) */
    int32_t s;                /* log2 leaves per work item for this group                   */
    uint32_t nsub;            /* work items (2^s-leaf subtrees) = 2^(depth - s)             */
    uint32_t pad;
    uint64_t table_off_v;     /* bin's first row, in uint4 units from EvalParams::table     */
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
    const GroupDesc *groups;  /* MODE_GROUPED(_ET): [key_groups] descriptors (else null)  */
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
};

/* Kernel modes. */
enum { MODE_FUSED = 0, MODE_EXPAND = 1, MODE_FRONTIER = 2, MODE_GROUPED = 3,
       MODE_FUSED_TMA = 4, /* MODE_FUSED with each work item's table rows staged into shared memory by
                             cp.async.bulk (16-column tables, non-AES PRFs, whole-warp key groups) */
       /* early-terminated keys (four table rows per leaf): the tree is over leaves, the table, the
        * leaf cache (EvalParams::n_local), the result and the shares (EvalParams::n) over rows; leaf
        * position p owns rows 4p..4p+3 of the device table */
       MODE_FUSED_ET = 5,  /* MODE_FUSED, nv = 4 or 8 */
       MODE_EXPAND_ET = 6, /* MODE_EXPAND: shares[key][4 * leaf + lane] */
       /* MODE_FUSED for AES at 16 columns with >= 4 keys per warp: the four lanes of a key quad split
        * each table row, lane L loading columns 4 (L & 3) .. +3, and the quad's leaf values travel by
        * SHFL instead, so a row costs the shared-memory data pipe one 16-byte load per lane, not four */
       MODE_FUSED_COLSPLIT = 7,
       /* MODE_GROUPED for early-terminated keys, nv = 4: GroupDesc::depth is the bin's leaf depth and
        * the bin's leaf position p owns its rows 4p..4p+3 */
       MODE_GROUPED_ET = 8,
       MODE_COUNT = 9 };

/* Threads per block (for a kernel mode: the column-split AES kernel runs 16 warps) / minimum blocks per SM of the kernel instantiated for
 * (prf, nv) where nv = uint4 (4 int32 columns) of a table row handled per pass:
 * 4, 8 or 16. */
int eval_threads(int prf, int nv, int mode);
int eval_min_blocks(int prf, int nv);

/* Shared-window address of the first dynamic shared memory byte (probed). */
cudaError_t probe_dynamic_smem_base(uint32_t *base, cudaStream_t stream);

/* Upload the AES T-table to this device's constant memory. */
cudaError_t upload_aes_table(const uint32_t *te0_256);

/* One pass of the fused evaluation (mode 0), the share expansion (mode 1) or the
 * frontier build (mode 2; nv must be 4 for modes 1 and 2).
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
 * from 44 seed bytes per key; keys in the reference wire format, [count][131] 128-bit slots each. */
cudaError_t launch_keygen(int prf, const int64_t *alphas, const uint8_t *seeds44, int64_t count, int depth, uint64_t n,
                          const uint32_t *te0, uint4 *keys_a, uint4 *keys_b, cudaStream_t stream);

/* Maximum dynamic shared memory the evaluation kernel may be given. */
cudaError_t eval_max_smem(int prf, int nv, int mode, int *bytes);

/* table[q][c] = stage[bitrev_bits(q)][c] for q < rows, c < cols; padded columns
 * [cols, stride) are left untouched (pre-zeroed).  The grid-stride helpers take the device's SM
 * count to cap their grids at a few waves.  With lane_bits = 2 (early-terminated contexts) rows
 * move in runs of four: table[4q + l] = stage[4 bitrev_bits(q) + l], rows = 4 * 2^bits. */
cudaError_t launch_permute_table(const int32_t *stage, int32_t *table, uint64_t rows, int bits,
                                 int cols, int stride, int sm_count, cudaStream_t stream);
cudaError_t launch_permute_table_et(const int32_t *stage, int32_t *table, uint64_t rows, int bits,
                                    int cols, int stride, int sm_count, cudaStream_t stream);

/* Row update of a live table (b200dpf_update_rows*): table row position(idx[j]) := rows[j] for
 * j < count, the last occurrence of a position winning.  Position of natural index i:
 *   bins == null   skip unless 0 <= i < n and (i & own_mask) == own_val;
 *                  else bitrev_depth(i >> shift)                      (whole table or one shard)
 *   bins != null   bin g = bins[j] (skip unless 0 <= g < nbins); skip unless 0 <= i < 2^bin_info[g].y;
 *                  else bin_info[g].x + bitrev_{bin_info[g].y}(i)     (grouped context)
 *   bins != null and lane_bits = 2 (early-terminated grouped context, .y = the bin's leaf depth):
 *                  skip unless 0 <= i < 4 << bin_info[g].y;
 *                  else bin_info[g].x + (bitrev_{bin_info[g].y}(i >> 2) << 2 | (i & 3))
 * Skipped entries are never written. */
struct UpdateParams {
    const int64_t *idx;       /* [count] natural indices                                      */
    const int32_t *bins;      /* [count] bin ids, or null                                     */
    const uint2 *bin_info;    /* [nbins] (first row, depth)                                   */
    int nbins;
    const int32_t *rows;      /* [count][cols] new rows                                       */
    int64_t count;            /* <= 2^31 - 1                                                  */
    int64_t n;
    uint32_t own_mask, own_val;
    int shift, depth;
    uint32_t table_rows;      /* rows of the device table: the skip marker, larger than every position */
    int lane_bits;            /* log2 rows per leaf: 0, or 2 on an early-terminated context, where
                                 row i < n belongs to leaf v = i >> 2, is owned when (v & own_mask)
                                 == own_val and goes to row 4 bitrev_depth(v >> shift) + (i & 3).
                                 (It fills the alignment gap before `table`: the struct's layout is
                                 that of the update kernels without it.)                          */
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

}  // namespace b200dpf
