"""dpf.DPF -- the reference's Python API (dpf.py:35-137) on the H100-native engine.

Same class, method names, argument meaning and exceptions as the reference, so
`sample.py` and `benchmark.py` written against it keep working:

    d = DPF(prf=DPF.PRF_AES128)
    k1, k2 = d.gen(index, n)        # client: two int32[524] CPU key tensors
    d.eval_init(table)              # server: upload [n, entry_size] table
    shares = d.eval_gpu([k1, ...])  # server: int32 [len(keys), entry_size] on the CPU

What differs is behind the boundary: `dpf_cpp` here is the pybind shim over
include/b200dpf.h (hand-written sm_90a kernels), tables may have any entry
size, batches may have any length (no pad-to-512 round trip, no pad-to-16
columns), and one process can own an entry-range shard of the table
(`DPF(prf, device=d, shard=(rank, count))`) whose partial results add mod 2^32.

The module-level test_* / *_perf helpers mirror the reference's self-tests
(dpf.py:139-356): same names and defaults, same pass criteria.
"""
import collections
import os
import random
import sys
import time

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

try:
    import dpf_cpp
except ImportError as exc:  # fail loudly: there is no Python/CPU stand-in for the kernels
    raise ImportError(
        "dpf_cpp extension not built (run `python gpu-dpf_b200/build.py`); "
        "the DPF engine has no fallback implementation: %s" % exc)


# What DPF does differently per kind of key (include/b200dpf.h): the dpf_cpp functions, whether explicit seeds
# are ChaCha20-DRBG bytes only (at least 44 per key) or may also select the reference's 32-bit mt19937
# generator, and the name in messages.  `gen` / `gen_batch` are the ChaCha20-DRBG generators.
# `id` is the kind's B200DPF_KIND_* (the trimmed contexts' kind argument).
_Kind = collections.namedtuple("_Kind", "name drbg_only gen gen_batch eval_cpu eval_init pack id")
_STANDARD = _Kind("standard", False, dpf_cpp.gen_secure, dpf_cpp.gen_batch_secure, dpf_cpp.eval_cpu,
                  dpf_cpp.eval_init_sharded, dpf_cpp.key_pack, 0)
_EARLY_TERMINATED = _Kind("early-terminated", True, dpf_cpp.gen_et, dpf_cpp.gen_batch_et, dpf_cpp.eval_cpu_et,
                          dpf_cpp.eval_init_et, dpf_cpp.key_pack_et, 1)
_XOR_SHARED = _Kind("XOR-shared", True, dpf_cpp.gen_xor, dpf_cpp.gen_batch_xor, dpf_cpp.eval_cpu_xor,
                    dpf_cpp.eval_init_xor, dpf_cpp.key_pack_xor, 2)


class DPF(object):

    PRF_CHACHA20 = dpf_cpp.PRF_CHACHA20
    PRF_DUMMY = dpf_cpp.PRF_DUMMY
    PRF_SALSA20 = dpf_cpp.PRF_SALSA20
    PRF_AES128 = dpf_cpp.PRF_AES128

    ENTRY_SIZE = dpf_cpp.ENTRY_SIZE
    BATCH_SIZE = dpf_cpp.BATCH_SIZE

    DEFAULT_PRF = dpf_cpp.PRF_AES128

    _PRF_NAMES = {
        dpf_cpp.PRF_CHACHA20: "CHACHA20",
        dpf_cpp.PRF_DUMMY: "DUMMY",
        dpf_cpp.PRF_SALSA20: "SALSA20",
        dpf_cpp.PRF_AES128: "AES128",
    }

    def __init__(self, prf=None, device=0, shard=(0, 1), allow_non_pow2=False, devices=None, axis="auto",
                 early_termination=False, xor=False, trim=False):
        # devices: None (one GPU: `device`), "all", or a list of device ids -- one process drives them all
        # (b200dpf_create_multi); axis "auto" | "entries" | "keys".  B200DPF_DEVICES / B200DPF_AXIS in the
        # environment set the defaults, so an unchanged `dpf.DPF()` caller (benchmark.py) can scale too.
        if devices is None and os.environ.get("B200DPF_DEVICES"):
            devices = os.environ["B200DPF_DEVICES"]
            axis = os.environ.get("B200DPF_AXIS", axis)
        if isinstance(devices, str):
            devices = dpf_cpp.parse_devices(devices)
        self.devices = list(devices) if devices is not None and len(devices) > 1 else None
        if devices is not None and len(devices) == 1:
            device = devices[0]
        self.axis = axis
        # allow_non_pow2: tables / domains whose size is not a power of two are padded with zero
        # rows up to the next one (a reference TODO, dpf.py:21; off by default so the reference's
        # "must be a power of two" errors stay as they are)
        self.allow_non_pow2 = allow_non_pow2
        self.buffers = None
        self.table_num_entries = None
        self.table_effective_entry_size = None
        self.table = None
        self.table_rows = None
        self.device = device
        self.shard = tuple(shard)
        self.prf_method = prf if prf is not None else self.DEFAULT_PRF
        self.prf_method_string = self._PRF_NAMES[self.prf_method]
        # early_termination: keys whose leaves carry four table rows each (include/b200dpf.h, b200dpf_gen_et):
        # about a quarter of the tree to expand.  Keys of the two kinds are not interchangeable.
        self.early_termination = bool(early_termination)
        if self.early_termination and self.devices:
            raise Exception("early_termination=True has no multi-device variant: use one device per DPF "
                            "(DPF(device=d, shard=(rank, count), early_termination=True))")
        # xor: two-server XOR PIR (include/b200dpf.h, b200dpf_gen_xor): each leaf carries 128 one-bit row shares,
        # and the two servers' results XOR (not add) to the selected row: eval_a ^ eval_b == table[k]
        self.xor = bool(xor)
        if self.xor and self.early_termination:
            raise Exception("xor=True and early_termination=True are different kinds of key: pass one of them")
        if self.xor and self.devices:
            raise Exception("xor=True has no multi-device variant: use one device per DPF "
                            "(DPF(device=d, shard=(rank, count), xor=True))")
        self.kind = _XOR_SHARED if self.xor else _EARLY_TERMINATED if self.early_termination else _STANDARD
        # trim: tables of any row count without padding to a power of two (include/b200dpf.h,
        # b200dpf_create_trimmed).  Row k is reached by an ordinary key of the kind for index
        # trimmed_alpha(k, n) over trimmed_domain(n) rows, which gen / gen_batch make from k and n.
        self.trim = bool(trim)
        if self.trim and self.devices:
            raise Exception("trim=True has no multi-device variant: a trimmed table lives on one GPU (DPF(device=d, trim=True))")
        if self.trim and self.shard != (0, 1):
            raise Exception("trim=True has no sharded variant: a trimmed context holds the whole table")
        self._trim_order = None

    # ---- client -----------------------------------------------------------
    def gen(self, k, n, seed=None, secure=None):
        """Two keys for the point function at index k over a domain of n (dpf.py:63-74).

        By default (no seed given) every random word comes from a ChaCha20 DRBG keyed with fresh
        os.urandom entropy.  The reference seeds std::mt19937 with 32 bits of its seed
        (dpf_wrapper.cu:52; its own TODO, dpf.py:65), so a server could enumerate the 2^32 possible
        generator states of a key it holds and recover the index: that generator is kept only
        for callers that pass an explicit `seed` (deterministic keys, bit-identical to the
        reference's for the same seed: golden and parity tests) and do not ask for secure=True."""
        if self.kind.drbg_only:
            # early-terminated and XOR-shared keys draw from the ChaCha20 DRBG only: explicit seeds are >= 44 bytes
            if secure is False:
                raise Exception("%s keys have no secure=False generator: pass >= 44 seed bytes or none" % self.kind.name)
            if seed is None:
                seed = os.urandom(44)
            if not isinstance(seed, (bytes, bytearray)) or len(seed) < 44:
                raise Exception("%s keys take a seed of at least 44 bytes" % self.kind.name)
            seed, secure = bytes(seed), True
        if secure is None:
            secure = seed is None
        if seed is None:
            seed = os.urandom(128)
        if self.trim:
            if not 0 <= k < n:
                raise Exception("k (%d), the selected row, must be in [0, n) with n (%d) the number of rows in the table" % (k, n))
            return (self.kind.gen if secure else dpf_cpp.gen)(dpf_cpp.trimmed_alpha(k, n, self.kind.id),
                                                              dpf_cpp.trimmed_domain(n, self.kind.id), seed, self.prf_method)
        if n & (n - 1) != 0 and not self.allow_non_pow2:
            raise Exception("Table num entries (%d) must be a power of two" % (n))
        if k >= n:
            raise Exception("k (%d), the selected element, must be less than n (%d), the number of entries in the table"
                            % (k, n))
        return (self.kind.gen if secure else dpf_cpp.gen)(k, _next_pow2(n), seed, self.prf_method)

    def gen_batch(self, indices, n, seeds=None, nthreads=0):
        """Keys for many indices at once: two int32 [B, 524] tensors (multi-threaded keygen).
        seeds=None: ChaCha20-DRBG keys from os.urandom entropy (44 bytes per key); explicit integer
        seeds select the reference's 32-bit mt19937 generator (deterministic, for tests).  With
        early_termination or xor, explicit seeds are bytes: 44 per key, concatenated.  With trim, n is any row
        count and each index a row < n."""
        idx = torch.as_tensor(list(indices), dtype=torch.int64)
        if self.trim:
            if idx.numel() and not (0 <= int(idx.min()) and int(idx.max()) < n):
                raise Exception("indices must be rows in [0, n) with n (%d) the number of rows in the table" % n)
            idx = torch.as_tensor([dpf_cpp.trimmed_alpha(int(r), n, self.kind.id) for r in idx], dtype=torch.int64)
            n = dpf_cpp.trimmed_domain(n, self.kind.id)
        if n & (n - 1) != 0:
            raise Exception("Table num entries (%d) must be a power of two" % (n))
        if self.kind.drbg_only:
            if seeds is None:
                seeds = os.urandom(44 * idx.numel())
            if not isinstance(seeds, (bytes, bytearray)) or len(seeds) != 44 * idx.numel():
                raise Exception("%s gen_batch takes seeds as bytes, 44 per key" % self.kind.name)
            return self.kind.gen_batch(idx, n, bytes(seeds), self.prf_method, nthreads)
        if idx.numel() and int(idx.max()) >= n:
            raise Exception("k (%d), the selected element, must be less than n (%d), the number of entries in the table"
                            % (int(idx.max()), n))
        if seeds is None:
            return self.kind.gen_batch(idx, n, os.urandom(44 * idx.numel()), self.prf_method, nthreads)
        return dpf_cpp.gen_batch(idx, n, torch.as_tensor(seeds, dtype=torch.int64), self.prf_method, nthreads)

    # ---- server -----------------------------------------------------------
    def eval_cpu(self, keys, one_hot_only=False):
        """CPU evaluation (dpf.py:76-86): share vectors, or shares @ table.  With xor: share bits (int32 0/1),
        or the XOR of the rows whose share bit is set."""
        if self.xor:
            return self._eval_cpu_xor(keys, one_hot_only)
        eval_one = self.kind.eval_cpu
        if one_hot_only:
            return self._rows(torch.stack([eval_one(k, self.prf_method) for k in keys]))
        if self.table is None:
            raise Exception("Must call `eval_init` before `eval_cpu` with one_hot_only=False")
        one_hots = self._rows(torch.stack([eval_one(k, self.prf_method) for k in keys]))
        return torch.matmul(one_hots, self.table)

    def _rows(self, shares):
        """Share vectors [B, domain] in row order: with trim, column r is the share of row r (index trimmed_alpha(r))."""
        if not self.trim:
            return shares
        if self.table is None:
            raise Exception("Must call `eval_init` before `eval_cpu` with trim=True: the row order depends on the table size")
        if self._trim_order is None:
            n = self.table.shape[0]
            self._trim_order = torch.as_tensor([dpf_cpp.trimmed_alpha(r, n, self.kind.id) for r in range(n)], dtype=torch.int64)
        return shares[:, self._trim_order]

    def _eval_cpu_xor(self, keys, one_hot_only):
        shifts = torch.arange(32, dtype=torch.int32)
        # packed words [B, n/32] -> bits [B, n]: row i is bit (i & 31) of word i >> 5
        bits = torch.stack([(self.kind.eval_cpu(k, self.prf_method).view(-1, 1) >> shifts) & 1 for k in keys])
        bits = self._rows(bits.reshape(len(keys), -1))
        if one_hot_only:
            return bits
        if self.table is None:
            raise Exception("Must call `eval_init` before `eval_cpu` with one_hot_only=False")
        # XOR of the selected rows, bit plane by bit plane: the parity of each plane's selected-row count
        table = self.table.to(torch.int32)
        sel = bits.to(torch.int64)
        out = torch.zeros((len(keys), table.shape[1]), dtype=torch.int32)
        for b in range(32):
            plane = ((table >> b) & 1).to(torch.int64)
            out |= ((torch.matmul(sel, plane) & 1).to(torch.int32) << b)
        return out

    def eval_init(self, table):
        """Upload the table (dpf.py:88-113).  Any entry size; no column padding."""
        if self.buffers is not None:
            dpf_cpp.eval_free(self.buffers)
            self.buffers = None
        if table.shape[0] < (1 if self.trim else 128):
            raise Exception("Table (%d) must have at least 128 elements" % table.shape[0])
        # the caller's row count: with allow_non_pow2 the rows beyond it are zero padding that updates may not touch
        self.table_rows = table.shape[0]
        # eval_cpu reads self.table; update_rows copies it before the first write, never writing the caller's tensor
        self._table_is_callers = True
        self._trim_order = None
        if table.shape[0] & (table.shape[0] - 1) != 0 and not self.trim:
            if not self.allow_non_pow2:
                raise Exception("Table num entries (%d) must be a power of two" % (table.shape[0]))
            table = _pad_rows_to_pow2(table)
            self._table_is_callers = False
        self.table = table
        self.table_num_entries = table.shape[0]
        self.table_effective_entry_size = table.shape[1]
        if self.trim:
            self.buffers = dpf_cpp.eval_init_trimmed(table, self.device, self.kind.id)
        elif self.devices:    # standard keys only: __init__ refuses the other kinds with devices
            self.buffers = dpf_cpp.eval_init_multi(table, self.devices, {"auto": 0, "entries": 1, "keys": 2}[self.axis])
        else:
            self.buffers = self.kind.eval_init(table, self.device, self.shard[0], self.shard[1])

    def update_rows(self, indices, rows):
        """Replace rows of the uploaded table in place: table[indices[j]] := rows[j] for natural indices (the
        numbering keys use; with trim, row numbers); when an index repeats, its last row wins.  `rows` [count, entry_size] is cast to
        int32 like eval_init's table.  Only the touched rows move: no re-upload, and `buffers` stays valid.

        CPU tensors (or lists) are applied synchronously.  CUDA tensors on the context's device are applied on
        the current torch stream, after every evaluation issued before and before every one issued after,
        without the host waiting for the update itself; the index range check before it does synchronise
        (one reduction read back), and so does keeping self.table in step when it lives on the CPU.
        self.table (what eval_cpu multiplies with) follows every update; the tensor passed to eval_init is
        copied on the first update and never written."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `update_rows`")
        idx, rows = _update_args(indices, rows, self.table_effective_entry_size)
        if idx.is_cuda != rows.is_cuda or (idx.is_cuda and (idx.device.index != self.device or rows.device.index != self.device)):
            raise Exception("indices and rows must both be CPU tensors or both CUDA tensors on cuda:%d" % self.device)
        if idx.is_cuda and self.devices:
            raise Exception("a multi-device DPF takes host rows (CPU tensors); device-resident updates are per GPU "
                            "(DPF(device=d, shard=(rank, count)) or sharded.ShardedDPF)")
        if idx.numel() and not bool(((idx >= 0) & (idx < self.table_rows)).all()):
            raise Exception("update index out of range [0, %d)" % self.table_rows)
        idx = idx.to(torch.int64).contiguous()
        rows = rows.to(torch.int32).contiguous()
        if idx.numel() == 0:
            return
        if idx.is_cuda:
            stream = torch.cuda.current_stream(idx.device).cuda_stream
            dpf_cpp.update_rows_device(idx.data_ptr(), rows.data_ptr(), idx.numel(), self.buffers, stream)
        else:
            dpf_cpp.update_rows(idx, rows, self.buffers)
        if self.table is not None:
            if self._table_is_callers:
                self.table = self.table.clone()
                self._table_is_callers = False
            uniq, inverse = torch.unique(idx, return_inverse=True)
            last = torch.full((uniq.numel(),), -1, dtype=torch.int64, device=idx.device).scatter_reduce_(
                0, inverse, torch.arange(idx.numel(), device=idx.device), "amax")
            self.table[uniq.to(self.table.device)] = rows[last].to(self.table.device, self.table.dtype)

    def eval_gpu(self, keys):
        """Evaluate a batch on the GPU (dpf.py:115-131): int32 [len(keys), entry_size] on the CPU.

        `keys` is a list of int32[524] tensors, or one int32 [B, 524] tensor."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `eval_gpu`")
        if isinstance(keys, torch.Tensor):
            if keys.is_cuda:        # keys already on the device: no staging at all
                return self.eval_gpu_device(keys.contiguous()).cpu()
            return dpf_cpp.eval_gpu_packed(keys.contiguous(), self.buffers, self.prf_method)
        if len(keys) == 0:
            return torch.zeros((0, self.table_effective_entry_size), dtype=torch.int32)
        return dpf_cpp.eval_gpu_list(list(keys), self.buffers, self.prf_method)

    def pack_keys(self, keys):
        """Compact wire form of a batch (24% to 56% smaller than int32[524] keys, depending on n): one
        contiguous uint8 tensor [B, 32 + 64*depth], pinned when CUDA is available, for eval_gpu_compact."""
        blobs = [self.kind.pack(k) for k in keys]
        t = torch.frombuffer(bytearray(b"".join(blobs)), dtype=torch.uint8).reshape(len(blobs), -1)
        return t.pin_memory() if torch.cuda.is_available() else t

    def eval_gpu_compact(self, packed):
        """eval_gpu for keys in the compact wire form (pack_keys): the packed bytes are what crosses PCIe."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `eval_gpu`")
        return dpf_cpp.eval_gpu_compact(packed.contiguous(), packed.shape[0], self.buffers, self.prf_method)

    def eval_gpu_device(self, keys_dev, out_dev=None, out_ptr=None, accumulate=False):
        """Device-resident, asynchronous variant: keys_dev int32 [B,524] CUDA tensor ->
        int32 [B, entry_size] CUDA tensor, enqueued on the current torch stream.
        accumulate=True adds into the destination instead of overwriting it (with xor: XORs into
        it); out_ptr may then be a raw (e.g. peer-mapped) device address."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `eval_gpu`")
        if self.devices:
            raise Exception("a multi-device DPF takes host keys (eval_gpu); device-resident evaluation is per GPU "
                            "(DPF(device=d, shard=(rank, count)) or sharded.ShardedDPF)")
        if not (keys_dev.is_cuda and keys_dev.dtype == torch.int32 and keys_dev.is_contiguous() and keys_dev.dim() == 2
                and keys_dev.shape[1] == 524 and keys_dev.device.index == self.device):
            raise Exception("keys_dev must be a contiguous int32 [B, 524] tensor on cuda:%d" % self.device)
        stream = torch.cuda.current_stream(keys_dev.device).cuda_stream
        if out_ptr is None:
            if out_dev is None:
                out_dev = torch.empty((keys_dev.shape[0], self.table_effective_entry_size), dtype=torch.int32,
                                      device=keys_dev.device)
            elif not (out_dev.is_cuda and out_dev.dtype == torch.int32 and out_dev.is_contiguous()
                      and out_dev.device == keys_dev.device
                      and tuple(out_dev.shape) == (keys_dev.shape[0], self.table_effective_entry_size)):
                raise Exception("out_dev must be a contiguous int32 [%d, %d] tensor on %s"
                                % (keys_dev.shape[0], self.table_effective_entry_size, keys_dev.device))
            out_ptr = out_dev.data_ptr()
        dpf_cpp.eval_gpu_device(keys_dev.data_ptr(), keys_dev.shape[0], self.buffers, self.prf_method,
                                out_ptr, stream, accumulate)
        return out_dev

    def eval_gpu_pipelined(self, batches, depth=2):
        """Server loop over a stream of batches (SURVEY.md section 8(f) rank 3): yields one CPU
        int32 [B, entry_size] tensor per input batch, in order.  Each batch is an int32 [B, 524]
        CPU tensor (pinned memory makes the copies truly asynchronous).  The host-to-device copy of
        batch i+1 and the device-to-host copy of batch i-1 run on their own streams while batch i
        is being evaluated, so in steady state only the kernel time is exposed."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `eval_gpu`")
        dev = torch.device("cuda", self.device)
        compute = torch.cuda.current_stream(dev)
        h2d, d2h = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        inflight = []                      # (out_host, done_event)

        def drain(limit):
            while len(inflight) > limit:
                out_host, done = inflight.pop(0)
                done.synchronize()
                yield out_host

        for keys in batches:
            keys = keys.contiguous()
            with torch.cuda.stream(h2d):
                keys_dev = keys.to(dev, non_blocking=True)
                copied = torch.cuda.Event()
                copied.record(h2d)
            compute.wait_event(copied)
            keys_dev.record_stream(compute)
            out_dev = self.eval_gpu_device(keys_dev)
            computed = torch.cuda.Event()
            computed.record(compute)
            with torch.cuda.stream(d2h):
                d2h.wait_event(computed)
                out_dev.record_stream(d2h)
                out_host = torch.empty(out_dev.shape, dtype=torch.int32, pin_memory=True)
                out_host.copy_(out_dev, non_blocking=True)
                done = torch.cuda.Event()
                done.record(d2h)
            inflight.append((out_host, done))
            yield from drain(depth)
        yield from drain(0)

    def expand_gpu_device(self, keys_dev, out_dev=None):
        """Share vectors on the GPU (the eval_cpu(one_hot_only=True) quantity): int32 [B, n] CUDA tensor.
        With xor the share bits come packed: int32 [B, n / 32], row i = bit (i & 31) of word i >> 5."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `expand_gpu_device`")
        if self.trim:
            raise Exception("expand_gpu_device has no trim=True variant: use eval_cpu(keys, one_hot_only=True) for share vectors "
                            "in row order")
        assert keys_dev.is_cuda and keys_dev.dtype == torch.int32 and keys_dev.is_contiguous()
        if out_dev is None:
            out_dev = torch.empty((keys_dev.shape[0], self.table_num_entries // (32 if self.xor else 1)), dtype=torch.int32,
                                  device=keys_dev.device)
        stream = torch.cuda.current_stream(keys_dev.device).cuda_stream
        dpf_cpp.expand_gpu_device(keys_dev.data_ptr(), keys_dev.shape[0], self.buffers, self.prf_method,
                                  out_dev.data_ptr(), stream)
        return out_dev

    def close(self):
        if self.buffers is not None:
            dpf_cpp.eval_free(self.buffers)
            self.buffers = None

    def __del__(self):
        # sample.py's server() builds a DPF per call and drops it: release the device table with the object
        # (the reference never frees unless eval_init is called again, dpf.py:93-94)
        try:
            self.close()
        except Exception:
            pass

    def __repr__(self):
        if self.buffers is None:
            return "DPF(_uninitialized_, prf_method=%s)" % self.prf_method_string
        return "DPF(entries=%d, entry_size=%d, prf_method=%s)" % (
            self.table_num_entries, self.table_effective_entry_size, self.prf_method_string)


class BinnedDPF(DPF):
    """Batch PIR (the paper's co-design front end, paper/experimental/batch_pir/batch_pir_optimization.py:84-87,
    210-218, which the reference only costs analytically): the table is split into bins, a query carries one DPF
    key per bin it touches, and the server evaluates all (bin, key) pairs of a batch of queries in ONE launch.

        d = BinnedDPF(prf=DPF.PRF_AES128)
        d.eval_init([bin0, bin1, ...])           # tables [n_g, entry_size], power-of-two n_g >= 2
        k1, k2 = d.gen_in_bin(g, index)          # keys for entry `index` of bin g
        shares = d.eval_gpu(keys, bins)          # int32 [len(keys), entry_size]

    With trim=True the bins may have any size n_g >= 1 (b200dpf_group_create_trimmed): gen_in_bin(g, index) makes
    the key of row `index` of bin g, and gen_queries_device maps its rows the same way.
    """

    def __init__(self, *args, **kwargs):
        if kwargs.get("early_termination"):
            raise Exception("BinnedDPF has no early-terminated variant (early_termination=True): use "
                            "dpf_cpp.group_init_et or b200dpf.GroupContext(early_termination=True)")
        if kwargs.get("xor"):
            raise Exception("BinnedDPF has no XOR-shared variant (xor=True): use "
                            "dpf_cpp.group_init_xor or b200dpf.GroupContext(xor=True)")
        super().__init__(*args, **kwargs)

    def eval_init(self, tables):
        if self.buffers is not None:
            dpf_cpp.eval_free(self.buffers)
            self.buffers = None
        tables = list(tables)
        for t in tables:
            if self.trim and t.shape[0] < 1:
                raise Exception("Table num entries (%d) must be at least 1" % (t.shape[0]))
            if not self.trim and (t.shape[0] & (t.shape[0] - 1) != 0 or t.shape[0] < 2):
                raise Exception("Table num entries (%d) must be a power of two" % (t.shape[0]))
        self.bin_sizes = [int(t.shape[0]) for t in tables]
        self.table = None
        self.table_num_entries = sum(self.bin_sizes)
        self.table_effective_entry_size = tables[0].shape[1]
        self.buffers = (dpf_cpp.group_init_trimmed(tables, self.device, self.kind.id) if self.trim
                        else dpf_cpp.group_init(tables, self.device))

    def gen_in_bin(self, g, k, seed=None, secure=False):
        return self.gen(k, self.bin_sizes[g], seed=seed, secure=secure)

    def eval_gpu(self, keys, bins):
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `eval_gpu`")
        if not isinstance(keys, torch.Tensor):
            if len(keys) == 0:
                return torch.zeros((0, self.table_effective_entry_size), dtype=torch.int32)
            keys = torch.stack(list(keys))
        return dpf_cpp.group_eval(keys.contiguous(), torch.as_tensor(bins), self.buffers, self.prf_method)

    def eval_gpu_device(self, keys_dev, bins, out_dev=None):
        """Device-resident, asynchronous variant of eval_gpu: keys_dev int32 [B, 524] CUDA tensor ->
        int32 [B, entry_size] CUDA tensor (out_dev, if given, is filled), enqueued on the current torch
        stream.  `bins` (one bin per key) stays on the host: the launch is planned from it without a sync."""
        if getattr(bins, "is_cuda", False):
            raise Exception("BinnedDPF.eval_gpu_device: bins must be on the host (a list, array or CPU tensor): the launch is planned from them, "
                            "and reading them from the device would need a synchronisation")
        if not (isinstance(keys_dev, torch.Tensor) and keys_dev.is_cuda and keys_dev.dtype == torch.int32
                and keys_dev.is_contiguous() and keys_dev.dim() == 2 and keys_dev.shape[1] == 524
                and keys_dev.device.index == self.device):
            raise Exception("BinnedDPF.eval_gpu_device: keys_dev must be a contiguous int32 [B, 524] tensor on cuda:%d" % self.device)
        bins = torch.as_tensor(bins)
        if bins.dim() != 1 or bins.numel() != keys_dev.shape[0] or bins.is_floating_point() or bins.dtype == torch.bool:
            raise Exception("BinnedDPF.eval_gpu_device: bins must be a 1-D integer tensor with one bin per key")
        if self.buffers is None:
            raise Exception("BinnedDPF.eval_gpu_device: must call `eval_init` first")
        shape = (keys_dev.shape[0], self.table_effective_entry_size)
        if out_dev is None:
            out_dev = torch.empty(shape, dtype=torch.int32, device=keys_dev.device)
        elif not (isinstance(out_dev, torch.Tensor) and out_dev.is_cuda and out_dev.dtype == torch.int32
                  and out_dev.is_contiguous() and out_dev.device == keys_dev.device and tuple(out_dev.shape) == shape):
            raise Exception("BinnedDPF.eval_gpu_device: out_dev must be a contiguous int32 [%d, %d] tensor on %s" % (shape + (keys_dev.device,)))
        stream = torch.cuda.current_stream(keys_dev.device).cuda_stream
        dpf_cpp.group_eval_device(keys_dev.data_ptr(), bins.to(torch.int32).contiguous(), keys_dev.shape[0], self.buffers,
                                  self.prf_method, out_dev.data_ptr(), stream)
        return out_dev

    def eval_gpu_device_bins(self, keys_dev, bins_dev, out_dev=None, bad_dev=None):
        """eval_gpu_device with the bins on the device too: keys_dev int32 [B, 524] and bins_dev int32 [B] CUDA
        tensors -> int32 [B, entry_size] CUDA tensor (out_dev, if given, is filled), planned on the GPU and enqueued
        on the current torch stream without any host wait.  A key whose bin is outside [0, nbins) gets a zero row;
        bad_dev, an int64 [1] CUDA tensor if given, receives the number of such keys."""
        name = "BinnedDPF.eval_gpu_device_bins"
        if not (isinstance(keys_dev, torch.Tensor) and keys_dev.is_cuda and keys_dev.dtype == torch.int32
                and keys_dev.is_contiguous() and keys_dev.dim() == 2 and keys_dev.shape[1] == 524
                and keys_dev.device.index == self.device):
            raise Exception("%s: keys_dev must be a contiguous int32 [B, 524] tensor on cuda:%d" % (name, self.device))
        if not (isinstance(bins_dev, torch.Tensor) and bins_dev.is_cuda and bins_dev.dtype == torch.int32
                and bins_dev.is_contiguous() and tuple(bins_dev.shape) == (keys_dev.shape[0],)
                and bins_dev.device == keys_dev.device):
            raise Exception("%s: bins_dev must be a contiguous int32 [%d] tensor on %s (one bin per key)"
                            % (name, keys_dev.shape[0], keys_dev.device))
        if bad_dev is not None and not (isinstance(bad_dev, torch.Tensor) and bad_dev.is_cuda and bad_dev.dtype == torch.int64
                                        and bad_dev.numel() == 1 and bad_dev.device == keys_dev.device):
            raise Exception("%s: bad_dev must be an int64 [1] tensor on %s" % (name, keys_dev.device))
        if self.buffers is None:
            raise Exception("%s: must call `eval_init` first" % name)
        shape = (keys_dev.shape[0], self.table_effective_entry_size)
        if out_dev is None:
            out_dev = torch.empty(shape, dtype=torch.int32, device=keys_dev.device)
        elif not (isinstance(out_dev, torch.Tensor) and out_dev.is_cuda and out_dev.dtype == torch.int32
                  and out_dev.is_contiguous() and out_dev.device == keys_dev.device and tuple(out_dev.shape) == shape):
            raise Exception("%s: out_dev must be a contiguous int32 [%d, %d] tensor on %s" % ((name,) + shape + (keys_dev.device,)))
        stream = torch.cuda.current_stream(keys_dev.device).cuda_stream
        dpf_cpp.group_eval_device_bins(keys_dev.data_ptr(), bins_dev.data_ptr(), keys_dev.shape[0], self.buffers, self.prf_method,
                                       out_dev.data_ptr(), 0 if bad_dev is None else bad_dev.data_ptr(), stream)
        return out_dev

    def eval_queries_device(self, keys_dev, out_dev=None):
        """Batch-PIR queries of one key per bin, device-resident and asynchronous: keys_dev is a CUDA tensor of
        Q queries, either int32 [Q, nbins, 524] wire-format keys (key g of a query for bin g) or uint8
        [Q, query_bytes] compact queries (the keys' key_pack forms back to back, dpf_cpp.group_query_bytes
        bytes); returns int32 [Q, nbins, entry_size] (out_dev, if given, is filled), enqueued on the current
        torch stream.  The launch plan depends on Q alone and is reused from one call of the same Q to the next."""
        name = "BinnedDPF.eval_queries_device"
        if self.buffers is None:
            raise Exception("%s: must call `eval_init` first" % name)
        nbins = len(self.bin_sizes)
        if not (isinstance(keys_dev, torch.Tensor) and keys_dev.is_cuda and keys_dev.is_contiguous()
                and keys_dev.device.index == self.device and keys_dev.dtype in (torch.int32, torch.uint8)):
            raise Exception("%s: keys_dev must be a contiguous CUDA tensor on cuda:%d, int32 [Q, %d, 524] or uint8 "
                            "[Q, query_bytes]" % (name, self.device, nbins))
        if keys_dev.dtype == torch.int32:
            compact = False
            if keys_dev.dim() != 3 or tuple(keys_dev.shape[1:]) != (nbins, 524):
                raise Exception("%s: int32 keys_dev must be [Q, %d, 524] (one wire-format key per bin per query), got %s"
                                % (name, nbins, tuple(keys_dev.shape)))
        else:
            compact = True
            qb = dpf_cpp.group_query_bytes(self.buffers)
            if keys_dev.dim() != 2 or keys_dev.shape[1] != qb:
                raise Exception("%s: uint8 keys_dev must be [Q, %d] (one compact query per row), got %s"
                                % (name, qb, tuple(keys_dev.shape)))
        shape = (keys_dev.shape[0], nbins, self.table_effective_entry_size)
        if out_dev is None:
            out_dev = torch.empty(shape, dtype=torch.int32, device=keys_dev.device)
        elif not (isinstance(out_dev, torch.Tensor) and out_dev.is_cuda and out_dev.dtype == torch.int32
                  and out_dev.is_contiguous() and out_dev.device == keys_dev.device and tuple(out_dev.shape) == shape):
            raise Exception("%s: out_dev must be a contiguous int32 [%d, %d, %d] tensor on %s" % ((name,) + shape + (keys_dev.device,)))
        stream = torch.cuda.current_stream(keys_dev.device).cuda_stream
        dpf_cpp.group_eval_queries_device(keys_dev.data_ptr(), keys_dev.shape[0], self.buffers, self.prf_method,
                                          out_dev.data_ptr(), stream, compact)
        return out_dev

    def gen_queries_device(self, indices_dev, seeds_dev=None, compact=True):
        """Both servers' batch-PIR queries, made on the GPU for the queries eval_queries_device takes (a load
        generator's or a benchmark's client side): indices_dev is an int64 [Q, nbins] CUDA tensor, the row of bin
        g that query q selects (taken mod the bin's size); seeds_dev a uint8 [Q, nbins, 44] CUDA tensor of key
        entropy, or None for os.urandom bytes.  Returns two CUDA tensors, uint8 [Q, query_bytes] compact queries
        (compact=True) or int32 [Q, nbins, 524] wire-format keys, enqueued on the current torch stream; key
        (q, g) is the one gen_in_bin(g, index, secure=True) makes from the same 44 seed bytes."""
        name = "BinnedDPF.gen_queries_device"
        if self.buffers is None:
            raise Exception("%s: must call `eval_init` first" % name)
        nbins = len(self.bin_sizes)
        if not (isinstance(indices_dev, torch.Tensor) and indices_dev.is_cuda and indices_dev.dtype == torch.int64
                and indices_dev.is_contiguous() and indices_dev.device.index == self.device
                and indices_dev.dim() == 2 and indices_dev.shape[1] == nbins):
            raise Exception("%s: indices_dev must be a contiguous int64 [Q, %d] tensor on cuda:%d" % (name, nbins, self.device))
        nq = indices_dev.shape[0]
        if seeds_dev is None:
            seeds_dev = torch.frombuffer(bytearray(os.urandom(44 * nq * nbins)), dtype=torch.uint8).reshape(nq, nbins, 44)
            seeds_dev = seeds_dev.to(indices_dev.device)
        elif not (isinstance(seeds_dev, torch.Tensor) and seeds_dev.is_cuda and seeds_dev.dtype == torch.uint8
                  and seeds_dev.is_contiguous() and seeds_dev.device == indices_dev.device
                  and tuple(seeds_dev.shape) == (nq, nbins, 44)):
            raise Exception("%s: seeds_dev must be a contiguous uint8 [%d, %d, 44] tensor on %s"
                            % (name, nq, nbins, indices_dev.device))
        if compact:
            shape, dtype = (nq, dpf_cpp.group_query_bytes(self.buffers)), torch.uint8
        else:
            shape, dtype = (nq, nbins, 524), torch.int32
        out_a = torch.empty(shape, dtype=dtype, device=indices_dev.device)
        out_b = torch.empty(shape, dtype=dtype, device=indices_dev.device)
        stream = torch.cuda.current_stream(indices_dev.device).cuda_stream
        dpf_cpp.group_gen_queries_device(indices_dev.data_ptr(), seeds_dev.data_ptr(), nq, self.buffers, self.prf_method,
                                         out_a.data_ptr(), out_b.data_ptr(), stream, compact)
        return out_a, out_b

    def update_rows(self, bins, indices, rows):
        """Replace rows of live bins: row indices[j] of bin bins[j] := rows[j] (the last occurrence of a
        (bin, index) pair wins); synchronous.  A bin or index out of range raises, and nothing is applied."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `update_rows`")
        idx, rows = _update_args(indices, rows, self.table_effective_entry_size)
        bins = torch.as_tensor(bins)
        if bins.dim() != 1 or bins.numel() != idx.numel() or bins.is_floating_point() or bins.dtype == torch.bool:
            raise Exception("bins must be a 1-D integer tensor with one bin per index")
        dpf_cpp.group_update_rows(bins.to(torch.int32).cpu().contiguous(), idx.to(torch.int64).cpu().contiguous(),
                                  rows.to(torch.int32).cpu().contiguous(), self.buffers)

    def __repr__(self):
        if self.buffers is None:
            return "BinnedDPF(_uninitialized_, prf_method=%s)" % self.prf_method_string
        return "BinnedDPF(bins=%d, entries=%d, entry_size=%d, prf_method=%s)" % (
            len(self.bin_sizes), self.table_num_entries, self.table_effective_entry_size, self.prf_method_string)


class BatchCodeDPF(BinnedDPF):
    """Any k rows of one table per query (include/b200dpf.h, b200dpf_batchcode_create): the server stores every row in
    3 of `nbins` bins, the client places its k rows in distinct bins (plan) and sends one key per bin, and the answers
    of the bins that hold the wanted rows reconstruct them.  With nbins about 1.5 k, every row is placed with high
    probability; a row that is not has slot -1 and found False.  Every kind of key (early_termination, xor).

        d = BatchCodeDPF(DPF.PRF_AES128, 0, nbins=48)
        d.eval_init(table)                                   # [n, entry_size]
        qa, qb, slots = d.gen_queries(wanted)                # wanted [Q, k] rows; keys int32 [Q, nbins, 524]
        rows, found = d.reconstruct(d.eval_queries_device(qa.cuda()), d.eval_queries_device(qb.cuda()), slots)

    `seed` is the public layout seed (None: random).  gen_in_bin, eval_gpu and the other BinnedDPF evaluations work on
    the bins as on a trimmed BinnedDPF."""

    def __init__(self, prf=None, device=0, nbins=None, seed=None, early_termination=False, xor=False):
        if nbins is None or int(nbins) < 1:
            raise Exception("BatchCodeDPF needs nbins >= 1 (about 1.5 times the rows wanted per query)")
        DPF.__init__(self, prf, device, early_termination=early_termination, xor=xor, trim=True)
        self.nbins = int(nbins)
        self.seed = int.from_bytes(os.urandom(8), "little") if seed is None else int(seed) & 0xFFFFFFFFFFFFFFFF
        self.n = None

    def use_layout(self, n):
        """Plan for a table of n rows without holding it: a client knows (n, nbins, seed), not the table.  eval_init
        does this too."""
        self.n = int(n)
        self.bin_sizes = [3 * ((self.n - j + self.nbins - 1) // self.nbins) for j in range(self.nbins)]

    def eval_init(self, table):
        if self.buffers is not None:
            dpf_cpp.eval_free(self.buffers)
            self.buffers = None
        table = torch.as_tensor(table)
        if table.dim() != 2:
            raise Exception("BatchCodeDPF.eval_init: table must be [n, entry_size]")
        self.buffers = dpf_cpp.batchcode_init(table, self.nbins, self.seed, self.device, self.kind.id)
        self.use_layout(table.shape[0])
        self.table = None
        self.table_num_entries = self.n
        self.table_effective_entry_size = int(table.shape[1])

    def _wanted(self, wanted, name):
        if self.n is None:
            raise Exception("BatchCodeDPF.%s: must call `eval_init` (or `use_layout`) first" % name)
        w = torch.as_tensor(wanted)
        if w.is_floating_point() or w.is_complex() or w.dtype == torch.bool or w.dim() not in (1, 2):
            raise Exception("BatchCodeDPF.%s: wanted must be an integer tensor [Q, k] (or [k] for one query)" % name)
        return w.reshape(1, -1) if w.dim() == 1 else w

    def plan(self, wanted):
        """The client's plan (b200dpf_batchcode_plan) of wanted rows [Q, k]: (alphas int64 [Q, nbins], the in-bin row
        to query in each bin; slots int32 [Q, k], the bin that answers each wanted row, or -1)."""
        w = self._wanted(wanted, "plan").to(torch.int64).cpu().contiguous()
        return tuple(dpf_cpp.batchcode_plan(self.n, self.nbins, self.seed, w))

    def gen_queries(self, wanted, seeds=None):
        """The host client: both servers' queries for wanted rows [Q, k], as int32 [Q, nbins, 524] wire-format keys
        (key g of query q for bin g, made by the kind's ChaCha20-DRBG keygen for trimmed_alpha(row, bin size)), and
        the slots of plan.  seeds: 44 bytes per key, Q * nbins keys in query-major order (None: os.urandom)."""
        alphas, slots = self.plan(wanted)
        nq = alphas.shape[0]
        if seeds is None:
            seeds = os.urandom(44 * nq * self.nbins)
        if not isinstance(seeds, (bytes, bytearray)) or len(seeds) != 44 * nq * self.nbins:
            raise Exception("BatchCodeDPF.gen_queries: seeds must be bytes, 44 per key (%d keys)" % (nq * self.nbins))
        qa = torch.zeros((nq, self.nbins, 524), dtype=torch.int32)
        qb = torch.zeros_like(qa)
        for size in sorted(set(self.bin_sizes)):         # the bins of one size share a key domain
            bins = [g for g in range(self.nbins) if self.bin_sizes[g] == size]
            idx = torch.as_tensor([dpf_cpp.trimmed_alpha(int(alphas[q, g]), size, self.kind.id)
                                   for q in range(nq) for g in bins], dtype=torch.int64)
            sd = b"".join(seeds[44 * (q * self.nbins + g):44 * (q * self.nbins + g + 1)] for q in range(nq) for g in bins)
            ka, kb = self.kind.gen_batch(idx, dpf_cpp.trimmed_domain(size, self.kind.id), sd, self.prf_method, 0)
            qa[:, bins] = ka.reshape(nq, len(bins), 524)
            qb[:, bins] = kb.reshape(nq, len(bins), 524)
        return qa, qb, slots

    def gen_queries_device(self, wanted_dev, seeds_dev=None, compact=True):
        """The device client for load generators: the plan of wanted_dev (an int64 [Q, k] CUDA tensor) on the GPU
        (b200dpf_batchcode_plan_device), then the keys on the GPU (BinnedDPF.gen_queries_device) from its alphas,
        all enqueued on the current torch stream.  Returns (qa, qb, slots): the two servers' queries in the format of
        `compact` and the slots int32 [Q, k] CUDA tensor, bit for bit those of plan."""
        name = "BatchCodeDPF.gen_queries_device"
        if self.buffers is None:
            raise Exception("%s: must call `eval_init` first" % name)
        if not (isinstance(wanted_dev, torch.Tensor) and wanted_dev.is_cuda and wanted_dev.dtype == torch.int64
                and wanted_dev.is_contiguous() and wanted_dev.dim() == 2 and wanted_dev.device.index == self.device):
            raise Exception("%s: wanted_dev must be a contiguous int64 [Q, k] tensor on cuda:%d" % (name, self.device))
        nq, k = wanted_dev.shape
        alphas = torch.empty((nq, self.nbins), dtype=torch.int64, device=wanted_dev.device)
        slots = torch.empty((nq, k), dtype=torch.int32, device=wanted_dev.device)
        stream = torch.cuda.current_stream(wanted_dev.device).cuda_stream
        dpf_cpp.batchcode_plan_device(wanted_dev.data_ptr(), nq, k, self.buffers, alphas.data_ptr(), slots.data_ptr(), stream)
        qa, qb = BinnedDPF.gen_queries_device(self, alphas, seeds_dev, compact)
        return qa, qb, slots

    def reconstruct(self, out_a, out_b, slots):
        """The wanted rows from both servers' answers (int32 [Q, nbins, entry_size], as eval_queries_device returns
        them) and the plan's slots [Q, k]: (rows int32 [Q, k, entry_size], found bool [Q, k]).  A row is a - b mod 2^32
        (XOR-shared keys: a ^ b) of its bin's answers; an unplaced row is zero and not found."""
        slots = torch.as_tensor(slots).to(device=out_a.device, dtype=torch.int64)
        if out_a.dim() != 3 or out_a.shape != out_b.shape or slots.dim() != 2 or slots.shape[0] != out_a.shape[0]:
            raise Exception("BatchCodeDPF.reconstruct: answers must be [Q, nbins, entry_size] and slots [Q, k]")
        found = slots >= 0
        idx = slots.clamp(min=0).unsqueeze(-1).expand(-1, -1, out_a.shape[2])
        a, b = torch.gather(out_a, 1, idx), torch.gather(out_b, 1, idx)
        rows = a ^ b if self.xor else a - b          # int32 wraps: the difference mod 2^32
        return rows * found.unsqueeze(-1).to(rows.dtype), found

    def update_rows(self, indices, rows):
        """Replace table rows in all three copies: row indices[j] := rows[j] (last occurrence wins); synchronous.  An
        index out of range raises, and nothing is applied."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `update_rows`")
        idx, rows = _update_args(indices, rows, self.table_effective_entry_size)
        dpf_cpp.batchcode_update_rows(idx.to(torch.int64).cpu().contiguous(), rows.to(torch.int32).cpu().contiguous(), self.buffers)

    def __repr__(self):
        if self.buffers is None:
            return "BatchCodeDPF(_uninitialized_, nbins=%d, prf_method=%s)" % (self.nbins, self.prf_method_string)
        return "BatchCodeDPF(entries=%d, nbins=%d, entry_size=%d, prf_method=%s)" % (
            self.n, self.nbins, self.table_effective_entry_size, self.prf_method_string)


class KeywordDPF(BinnedDPF):
    """A value by its 64-bit keyword in one query (include/b200dpf.h, b200dpf_kwpir_create): the server places each
    (keyword, value) item in one of three cuckoo hash tables of m slots, the client sends one key per table for its
    keyword's three candidate rows, and the answer whose stored keyword matches is the value; an absent keyword comes
    back zero with found False.  Every kind of key (early_termination, xor).

        d = KeywordDPF(DPF.PRF_AES128, 0)
        d.eval_init(keywords, values)                        # uint64 [n], int32 [n, E]
        qa, qb = d.gen_queries(query_keywords)               # keys int32 [Q, 3, 524]
        vals, found = d.reconstruct(d.eval_queries_device(qa.cuda()), d.eval_queries_device(qb.cuda()), query_keywords)

    m = ceil(expansion * n / 3) slots per table.  `seed` is the public layout seed (None: random); when a placement
    does not finish, eval_init retries seed + 1, seed + 2, ... (TRIES seeds in all) and `seed` is the one it ended
    with.  Keywords are uint64 (numpy arrays or Python ints) or int64 tensors holding their bits; keyword 2^64 - 1 is
    reserved.  The bins have value_size + 2 columns (the tag), so eval_queries_device returns [Q, 3, value_size + 2]."""

    TRIES = 8

    def __init__(self, prf=None, device=0, seed=None, expansion=1.3, early_termination=False, xor=False):
        if not expansion >= 1.0:
            raise Exception("KeywordDPF needs expansion >= 1 (3m slots for n items; 1.3 by default)")
        DPF.__init__(self, prf, device, early_termination=early_termination, xor=xor, trim=True)
        self.seed = int.from_bytes(os.urandom(8), "little") if seed is None else int(seed) & 0xFFFFFFFFFFFFFFFF
        self.expansion = float(expansion)
        self.n = self.m = self.value_size = None

    def use_layout(self, n, m, seed):
        """Locate keywords for a table of n items in 3 tables of m slots under `seed` without holding it: a client
        knows (n, m, seed), not the items.  eval_init does this too."""
        self.n, self.m, self.seed = int(n), int(m), int(seed) & 0xFFFFFFFFFFFFFFFF
        self.bin_sizes = [self.m] * 3

    def eval_init(self, keywords, values):
        if self.buffers is not None:
            dpf_cpp.eval_free(self.buffers)
            self.buffers = None
        kw = _keyword_tensor(keywords, "KeywordDPF.eval_init")
        values = torch.as_tensor(values)
        if values.dim() != 2 or values.shape[0] != kw.shape[0]:
            raise Exception("KeywordDPF.eval_init: values must be [n, value_size] with one row per keyword")
        n = int(kw.shape[0])
        m = max(-(-n // 3), int(np.ceil(self.expansion * n / 3)))
        for t in range(self.TRIES):
            seed = (self.seed + t) & 0xFFFFFFFFFFFFFFFF
            buffers = dpf_cpp.kwpir_init(kw, values, m, seed, self.device, self.kind.id)
            if buffers:
                break
        else:
            raise Exception("KeywordDPF.eval_init: the placement of %d items in 3 x %d slots did not finish for seeds %d..%d; "
                            "use a larger expansion" % (n, m, self.seed, seed))
        self.buffers = buffers
        self.use_layout(n, m, seed)
        self.value_size = int(values.shape[1])
        self.table = None
        self.table_num_entries = 3 * m
        self.table_effective_entry_size = self.value_size + 2

    def _need_layout(self, name):
        if self.m is None:
            raise Exception("KeywordDPF.%s: must call `eval_init` (or `use_layout`) first" % name)

    def plan(self, keywords):
        """The in-bin rows int64 [Q, 3] to query for keywords [Q] (b200dpf_kwpir_locate): row c is h_c(keyword)."""
        self._need_layout("plan")
        return dpf_cpp.kwpir_locate(self.m, self.seed, _keyword_tensor(keywords, "KeywordDPF.plan").cpu().contiguous())

    def gen_queries(self, keywords, seeds=None):
        """The host client: both servers' queries for keywords [Q], as int32 [Q, 3, 524] wire-format keys (key c of
        query q for bin c, made by the kind's ChaCha20-DRBG keygen for trimmed_alpha(h_c(keyword), m)).  seeds: 44
        bytes per key, 3Q keys in query-major order (None: os.urandom)."""
        alphas = self.plan(keywords)
        nq = alphas.shape[0]
        if seeds is None:
            seeds = os.urandom(44 * 3 * nq)
        if not isinstance(seeds, (bytes, bytearray)) or len(seeds) != 44 * 3 * nq:
            raise Exception("KeywordDPF.gen_queries: seeds must be bytes, 44 per key (%d keys)" % (3 * nq))
        idx = torch.as_tensor([dpf_cpp.trimmed_alpha(int(a), self.m, self.kind.id) for a in alphas.reshape(-1).tolist()],
                              dtype=torch.int64)
        ka, kb = self.kind.gen_batch(idx, dpf_cpp.trimmed_domain(self.m, self.kind.id), bytes(seeds), self.prf_method, 0)
        return ka.reshape(nq, 3, 524), kb.reshape(nq, 3, 524)

    def gen_queries_device(self, keywords_dev, seeds_dev=None, compact=True):
        """The device client for load generators: the rows of keywords_dev (an int64 [Q] CUDA tensor of the keywords'
        bits) on the GPU (b200dpf_kwpir_plan_device), then the keys on the GPU (BinnedDPF.gen_queries_device), all
        enqueued on the current torch stream.  Returns (qa, qb), the two servers' queries in the format of `compact`."""
        name = "KeywordDPF.gen_queries_device"
        if self.buffers is None:
            raise Exception("%s: must call `eval_init` first" % name)
        if not (isinstance(keywords_dev, torch.Tensor) and keywords_dev.is_cuda and keywords_dev.dtype in (torch.int64, torch.uint64)
                and keywords_dev.is_contiguous() and keywords_dev.dim() == 1 and keywords_dev.device.index == self.device):
            raise Exception("%s: keywords_dev must be a contiguous int64 [Q] tensor on cuda:%d" % (name, self.device))
        nq = keywords_dev.shape[0]
        alphas = torch.empty((nq, 3), dtype=torch.int64, device=keywords_dev.device)
        stream = torch.cuda.current_stream(keywords_dev.device).cuda_stream
        dpf_cpp.kwpir_plan_device(keywords_dev.data_ptr(), nq, self.buffers, alphas.data_ptr(), stream)
        return BinnedDPF.gen_queries_device(self, alphas, seeds_dev, compact)

    def reconstruct(self, out_a, out_b, keywords):
        """The values of keywords [Q] from both servers' answers (int32 [Q, 3, value_size + 2], as eval_queries_device
        returns them): (values int32 [Q, value_size], found bool [Q]).  A bin's row is a - b mod 2^32 (XOR-shared keys:
        a ^ b); the value is that of the bin whose tag is keyword + 1, and zero with found False when none is."""
        self._need_layout("reconstruct")
        e = self.value_size if self.value_size is not None else out_a.shape[-1] - 2
        kw = _keyword_tensor(keywords, "KeywordDPF.reconstruct").to(out_a.device)
        if out_a.dim() != 3 or out_a.shape != out_b.shape or tuple(out_a.shape[1:]) != (3, e + 2) or kw.shape[0] != out_a.shape[0]:
            raise Exception("KeywordDPF.reconstruct: answers must be [Q, 3, %d] and keywords [Q]" % (e + 2))
        rows = out_a ^ out_b if self.xor else out_a - out_b          # int32 wraps: the difference mod 2^32
        tag = kw.unsqueeze(1) + 1                                     # int64 wraps: keyword 2^64 - 1 has tag 0, never found
        lo = rows[..., e].to(torch.int64) & 0xFFFFFFFF
        hi = rows[..., e + 1].to(torch.int64) & 0xFFFFFFFF
        match = (lo == (tag & 0xFFFFFFFF)) & (hi == ((tag >> 32) & 0xFFFFFFFF)) & (tag != 0)
        values = torch.where(match.unsqueeze(-1), rows[..., :e], 0).sum(dim=1).to(torch.int32)
        return values, match.any(dim=1)

    def update(self, keywords, values):
        """Replace the values of present keywords: the value of keywords[j] := values[j] (last occurrence wins);
        synchronous.  A keyword that is not in the table raises, and nothing is applied."""
        if self.buffers is None:
            raise Exception("Must call `eval_init` before `update`")
        kw = _keyword_tensor(keywords, "KeywordDPF.update")
        values = torch.as_tensor(values)
        if values.dim() != 2 or values.shape[0] != kw.shape[0] or values.shape[1] != self.value_size:
            raise Exception("KeywordDPF.update: values must be [%d, %d] (one value per keyword)" % (kw.shape[0], self.value_size))
        dpf_cpp.kwpir_update(kw.cpu().contiguous(), values.to(torch.int32).cpu().contiguous(), self.buffers)

    def __repr__(self):
        if self.buffers is None:
            return "KeywordDPF(_uninitialized_, prf_method=%s)" % self.prf_method_string
        return "KeywordDPF(items=%d, m=%d, value_size=%d, prf_method=%s)" % (self.n, self.m, self.value_size, self.prf_method_string)


def _keyword_tensor(keywords, name):
    """keywords as a 1-D int64 tensor holding the uint64 keywords' bits (a tensor stays on its device)"""
    if isinstance(keywords, torch.Tensor):
        if keywords.dim() != 1 or keywords.is_floating_point() or keywords.is_complex() or keywords.dtype == torch.bool:
            raise Exception("%s: keywords must be a 1-D integer tensor or array of uint64 keywords" % name)
        return keywords.view(torch.int64) if keywords.dtype == torch.uint64 else keywords.to(torch.int64)
    a = keywords if isinstance(keywords, np.ndarray) else np.asarray(keywords, dtype=object)   # Python ints stay exact
    if a.dtype == object and a.ndim == 1 and all(isinstance(x, (int, np.integer)) for x in a):
        a = np.array([int(x) & 0xFFFFFFFFFFFFFFFF for x in a], np.uint64)
    if a.ndim != 1 or a.dtype.kind not in "iu":
        raise Exception("%s: keywords must be a 1-D integer tensor or array of uint64 keywords" % name)
    return torch.from_numpy(np.ascontiguousarray(a.astype(np.uint64).view(np.int64)))


def _next_pow2(n):
    return 1 << max(1, (n - 1).bit_length())


def _update_args(indices, rows, entry_size):
    """Shape and dtype checks of an update, before anything reaches the extension."""
    idx = torch.as_tensor(indices)
    rows = torch.as_tensor(rows)
    if idx.dim() != 1 or idx.is_floating_point() or idx.is_complex() or idx.dtype == torch.bool:
        raise Exception("indices must be a 1-D integer tensor")
    if rows.dim() != 2 or rows.shape[0] != idx.shape[0] or rows.shape[1] != entry_size:
        raise Exception("rows must be [%d, %d] (one row of entry_size columns per index), got %s"
                        % (idx.shape[0], entry_size, list(rows.shape)))
    if rows.is_complex() or rows.dtype == torch.bool:
        raise Exception("rows must be a real-valued tensor (cast to int32 like eval_init's table)")
    return idx, rows


def _pad_rows_to_pow2(table):
    """Zero rows up to the next power of two: they contribute nothing to any inner product."""
    pad = _next_pow2(table.shape[0]) - table.shape[0]
    return torch.cat([table, torch.zeros((pad, table.shape[1]), dtype=table.dtype, device=table.device)])


# ---------------------------------------------------------------------------
# self-tests and perf helpers, mirroring dpf.py:139-356 of the reference
# ---------------------------------------------------------------------------

def _gen_keys(dpf, batch, N):
    k1s, k2s, indices = [], [], []
    for _ in range(batch):
        indx = random.randint(0, N - 1)
        indices.append(indx)
        k1, k2 = dpf.gen(indx, N)
        k1s.append(k1)
        k2s.append(k2)
    return k1s, k2s, indices


def _index_table(N, cols=16, dtype=torch.int32):
    return (torch.arange(N).reshape(N, 1) * cols + torch.arange(cols).reshape(1, cols)).to(dtype)


def test_cpu_dpf_one_hot(N=1024):
    dpf = DPF()
    K = 42
    k1, k2 = dpf.gen(K, N)
    v1 = dpf.eval_cpu([k1], one_hot_only=True)
    v2 = dpf.eval_cpu([k2], one_hot_only=True)
    rec = (v1 - v2).numpy()
    gt = np.zeros(rec.shape)
    gt[:, K] = 1
    assert np.linalg.norm(rec - gt) <= 1e-8
    print("Pass CPU (one-hot only) check.")


def test_cpu_dpf(N=1024):
    dpf = DPF()
    k1s, k2s, gt_indices = _gen_keys(dpf, 64, N)
    dpf.table = _index_table(N)   # CPU-only: no device upload needed for eval_cpu
    a = dpf.eval_cpu(k1s)
    b = dpf.eval_cpu(k2s)
    rec = (a - b).numpy()
    gt = dpf.table[gt_indices, :].numpy()
    assert np.linalg.norm(rec - gt) <= 1e-8
    print("Pass CPU check.")


def test_gpu_dpf(N=8192):
    dpf = DPF()
    k1s, k2s, gt_indices = _gen_keys(dpf, 64, N)
    table = _index_table(N, dtype=torch.float32)   # the reference feeds a float table here
    dpf.eval_init(table)
    a = dpf.eval_gpu(k1s)
    b = dpf.eval_gpu(k2s)
    rec = (a - b).numpy()
    gt = table[gt_indices, :].numpy()
    assert np.linalg.norm(rec - gt) <= 1e-8
    print("Pass GPU check.")


def test_gpu_dpf_nopad(N=8192, batch=42, entrysize=13):
    dpf = DPF()
    k1s, k2s, gt_indices = _gen_keys(dpf, batch, N)
    table = torch.randint(2 ** 31, (N, entrysize)).int()
    dpf.eval_init(table)
    a = dpf.eval_gpu(k1s)
    b = dpf.eval_gpu(k2s)
    rec = (a - b).numpy()
    gt = table[gt_indices, :].numpy()
    assert np.linalg.norm(rec - gt) <= 1e-8
    print("Pass GPU (nopad) check.")


def test_gpu_dpf_sweep():
    for n in [128, 256, 512, 1024, 8192]:
        test_gpu_dpf_nopad(n, batch=random.randint(1, dpf_cpp.BATCH_SIZE * 5 - 1), entrysize=random.randint(1, 16 - 1))
    print("Pass GPU (sweep) check.")


def _perf(kind, N, batch, entrysize, prf):
    dpf = DPF(prf=prf)
    k1s, _, _ = _gen_keys(dpf, batch, N)
    table = torch.rand(N, entrysize).int()
    dpf.eval_init(table)
    fn = dpf.eval_gpu if kind == "gpu" else dpf.eval_cpu
    tstart = time.time()
    reps = 10
    for _ in range(reps):
        fn(k1s)
    elapsed = time.time() - tstart
    dpfs_per_sec = batch * reps / elapsed
    keysize = np.prod(k1s[0].shape) * 4
    print("%s Key Size: %d bytes, Perf: %d dpfs/sec" % (dpf, keysize, dpfs_per_sec))
    return dpfs_per_sec


def test_gpu_dpf_perf(N=2048, batch=dpf_cpp.BATCH_SIZE, entrysize=16, prf=DPF.DEFAULT_PRF):
    return _perf("gpu", N, batch, entrysize, prf)


def test_cpu_dpf_perf(N=2048, batch=dpf_cpp.BATCH_SIZE, entrysize=16, prf=DPF.DEFAULT_PRF):
    return _perf("cpu", N, batch, entrysize, prf)


if __name__ == "__main__":
    random.seed(time.time())
    test_cpu_dpf()
    test_cpu_dpf_one_hot()
    test_gpu_dpf()
    test_gpu_dpf_nopad()
    test_gpu_dpf_sweep()
    test_gpu_dpf_perf()
