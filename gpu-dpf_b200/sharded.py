"""One table across the GPUs of a box: one process per GPU (torchrun), two axes.

The reference is single-GPU (SURVEY.md section 2.2).

axis="entries" (default) -- entry-range sharding.  A DPF evaluation is a sum over
leaves, so disjoint leaf ranges give partial sums that add mod 2^32: rank r of
G = 2^g owns the GGM subtree under the depth-g node with breadth-first index r
(natural indices i with bitrev_g(i mod G) == r), holds only those n/G table rows,
evaluates EVERY key over its subtree, and the [B, E] int32 partials are reduced
to rank 0.  Two reductions are available:
    reduce="nccl"   one dist.reduce(SUM, int32) over NVLink (wrapping int32 add is
                    exactly the required arithmetic);
    reduce="fused"  no collective kernel at all: every rank's evaluation kernel adds
                    its partials straight into rank 0's result buffer through an
                    NVLink peer mapping (torch symmetric memory), i.e. the kernel's
                    red.global.add.u32 epilogue IS the reduction; two symmetric-
                    memory barriers order the clearing and the consumption.
axis="keys" -- replicas: every rank holds the whole table and evaluates a
contiguous slice of the batch; results are gathered on rank 0.  No arithmetic
crosses GPUs; right for small n where a shard would be tiny.

    dist.init_process_group("nccl")            # torchrun, one rank per GPU
    d = ShardedDPF(prf=DPF.PRF_AES128)         # device = LOCAL_RANK
    d.eval_init(table)                         # every rank passes the same table
    out = d.eval_gpu(keys)                     # rank 0: int32 [B, E] CPU tensor; others: None
"""
import os

import torch
import torch.distributed as dist


def shard_indices(n, rank, world):
    """Natural table indices owned by `rank`, in the breadth-first leaf order they are
    stored in on the device: position q of the shard holds index
    bitrev_{d-g}(q) * G + bitrev_g(rank).  (Pure index math; used by the tests.)"""
    d = n.bit_length() - 1
    g = world.bit_length() - 1
    assert 1 << d == n and 1 << g == world and world <= n // 2

    def brev(v, bits):
        r = 0
        for i in range(bits):
            r |= ((v >> i) & 1) << (bits - 1 - i)
        return r

    c = brev(rank, g)
    return [brev(q, d - g) * world + c for q in range(n // world)]


def key_slice(nkeys, rank, world):
    """[begin, end) of the batch evaluated by `rank` on the keys axis."""
    per = (nkeys + world - 1) // world
    return min(rank * per, nkeys), min((rank + 1) * per, nkeys)


class ShardedDPF(object):
    """dpf.DPF semantics over a process group; rank 0 receives the result."""

    # axis="auto": below this table size a shard is too small to keep a GPU busy and the partial-sum
    # reduce + the upload of every key to every rank dominate; the batch is split by keys instead
    AUTO_KEYS_MAX_N = 1 << 18

    def __init__(self, prf=None, group=None, device=None, axis="entries", reduce="nccl", early_termination=False,
                 xor=False):
        if early_termination:
            raise Exception("ShardedDPF has no early-terminated variant; a single-process shard is "
                            "dpf.DPF(shard=(rank, count), early_termination=True)")
        if xor:
            raise Exception("ShardedDPF has no XOR-shared variant; a single-process shard is "
                            "dpf.DPF(shard=(rank, count), xor=True), whose results XOR together")
        assert axis in ("entries", "keys", "auto") and reduce in ("nccl", "fused")
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        if axis == "entries" and self.world & (self.world - 1):
            raise Exception("number of shards (%d) must be a power of two" % self.world)
        if axis == "auto" and self.world & (self.world - 1):
            axis = "keys"
        self.device = int(os.environ.get("LOCAL_RANK", self.rank)) if device is None else device
        self.axis = axis
        self.reduce = reduce if self.world > 1 else "nccl"
        self._dpf = None
        self.prf = prf
        self.entry_size = None
        self.n = None
        self._symm = None        # (tensor, handle, rank-0 base pointer) for reduce="fused"
        self._keys_axis_buffers = None

    def eval_init(self, table):
        self.n, self.entry_size = table.shape[0], table.shape[1]
        import dpf
        if self.axis == "auto":
            self.axis = "keys" if (self.n <= self.AUTO_KEYS_MAX_N or self.world > self.n // 2) else "entries"
        shard = (self.rank, self.world) if self.axis == "entries" else (0, 1)
        self._dpf = dpf.DPF(prf=self.prf, device=self.device, shard=shard)
        self._dpf.eval_init(table)
        return self

    def update_rows(self, indices, rows):
        """table[indices[j]] := rows[j] on every rank (dpf.DPF.update_rows).  Every rank passes the same list,
        as with eval_init: an entry-range shard applies the rows it owns, a keys-axis replica applies all."""
        if self._dpf is None:
            raise Exception("Must call `eval_init` before `update_rows`")
        self._dpf.update_rows(indices, rows)

    # -- fused reduction plumbing ------------------------------------------------
    def _symm_buffer(self, nkeys):
        import torch.distributed._symmetric_memory as symm_mem
        need = nkeys * self.entry_size
        if self._symm is None or self._symm[0].numel() < need:
            dev = torch.device("cuda", self.device)
            t = symm_mem.empty(max(need, 1 << 16), dtype=torch.int32, device=dev)
            grp = self.group if self.group is not None else dist.group.WORLD
            hdl = symm_mem.rendezvous(t, grp.group_name)
            self._symm = (t, hdl, int(hdl.buffer_ptrs[0]))
        return self._symm

    # -- device-resident path (benchmarks, servers that keep keys on the GPU) --
    def eval_gpu_device(self, keys_dev, out_dev=None):
        """This rank's work on its stream, then the cross-GPU step.  Returns the device tensor
        holding the complete [B, E] result on rank 0 once the stream is synchronised."""
        nkeys = keys_dev.shape[0]
        if self.axis == "keys":
            # every rank evaluates its slice straight into its row block of one [world*per, E] buffer;
            # rank 0 gathers the blocks in place (buffers are kept between calls: at small n a step is
            # ~0.2 ms and fresh allocations would show)
            b, e = key_slice(nkeys, self.rank, self.world)
            per = (nkeys + self.world - 1) // self.world
            dev = keys_dev.device
            bufs = self._keys_axis_buffers
            # NCCL: one all-gather kernel (a gather is a batch of point-to-point sends with twice the latency;
            # the [B, E] result is a few KiB, so every rank receiving it costs nothing); gloo: a plain gather
            use_all_gather = dist.get_backend(self.group) == "nccl"
            if bufs is None or bufs[0] != (per, dev):
                mine = torch.zeros((per, self.entry_size), dtype=torch.int32, device=dev)
                need_full = self.rank == 0 or use_all_gather
                full = torch.empty((self.world * per, self.entry_size), dtype=torch.int32, device=dev) if need_full else None
                chunks = list(full.split(per)) if self.rank == 0 else None
                bufs = self._keys_axis_buffers = ((per, dev), mine, full, chunks)
            _, mine, full, chunks = bufs
            if e > b:
                self._dpf.eval_gpu_device(keys_dev[b:e], mine[:e - b])
            if use_all_gather:
                dist.all_gather_into_tensor(full, mine, group=self.group)
            else:
                dist.gather(mine, chunks, dst=0, group=self.group)
            if self.rank == 0:
                if out_dev is not None:
                    out_dev.copy_(full[:nkeys])
                    return out_dev
                return full[:nkeys]
            return None
        if self.world > 1 and self.reduce == "fused":
            t, hdl, root_ptr = self._symm_buffer(nkeys)
            view = t[:nkeys * self.entry_size].view(nkeys, self.entry_size)
            if self.rank == 0:
                view.zero_()
            hdl.barrier(channel=0)                 # destination cleared before anyone adds
            self._dpf.eval_gpu_device(keys_dev, out_ptr=root_ptr, accumulate=True)
            hdl.barrier(channel=1)                 # every rank's adds have landed
            if self.rank != 0:
                return None
            # the symmetric buffer is reused (and re-zeroed) by the next call: hand the caller a tensor
            # it owns, like the NCCL path does
            if out_dev is None:
                return view.clone()
            out_dev.copy_(view)
            return out_dev
        out_dev = self._dpf.eval_gpu_device(keys_dev, out_dev)
        return self._reduce_to_rank0(out_dev)

    # -- host-buffer path (the dpf.DPF.eval_gpu contract) --
    def eval_gpu(self, keys):
        if isinstance(keys, torch.Tensor):
            packed = keys.contiguous()
        else:
            packed = torch.stack(list(keys))
        self._check_keys(packed)
        out = self._evaluate_and_combine(packed)
        return out.cpu() if self.rank == 0 else None

    def _check_keys(self, packed):
        """The device-resident path takes the tree depth from the context, not from the key: refuse
        keys made for another domain size here, as DPF.eval_gpu does (slot 130 = n, slot 0 = depth)."""
        if packed.dtype != torch.int32 or packed.dim() != 2 or packed.shape[1] != 524:
            raise Exception("keys must be int32 [B, 524]")
        if self.n is None or packed.shape[0] == 0:
            return
        n_lo, depth = packed[:, 130 * 4], packed[:, 0]
        n_word = self.n if self.n < 2 ** 31 else self.n - 2 ** 32
        if not bool(((n_lo == n_word) & (depth == self.n.bit_length() - 1)).all()):
            raise RuntimeError("a key was generated for a different table size than n=%d" % self.n)

    def _evaluate_and_combine(self, packed):
        """This rank's evaluation on its GPU plus the cross-rank step; the tensor returned on
        rank 0 holds the complete result.  (The seam the CPU process-group tests override.)"""
        dev = torch.device("cuda", self.device)
        keys_dev = packed.to(dev, non_blocking=True)
        out_dev = self.eval_gpu_device(keys_dev)
        if self.rank != 0:
            torch.cuda.current_stream(dev).synchronize()
        return out_dev

    def _reduce_to_rank0(self, part):
        """Wrapping int32 sum of the per-shard partials onto rank 0."""
        if self.world > 1:
            dist.reduce(part, dst=0, op=dist.ReduceOp.SUM, group=self.group)
        return part

    def close(self):
        if self._dpf is not None:
            self._dpf.close()
