"""Concurrent use of one GPU (include/b200dpf.h, "Threading"), every result compared bit for bit with an oracle
computed on the host before any thread starts:

  * test_independent_contexts_on_threads: workers on their own host threads, each owning a context (standard,
    early-terminated and XOR-shared plain contexts, a trimmed one, a grouped one, one of 160 columns and a
    dpf.DPF object), run a fixed script of rounds through every entry point while another thread generates keys
    on the GPU and another creates and destroys contexts.  Three workers launch the same ChaCha20 kernel with
    different dynamic shared memory at the same time: a kernel's shared-memory ceiling is process-wide, so one
    context must never shrink it under another's launch;
  * test_one_context_many_streams: one context, evaluations rotating over three streams with no host
    synchronisation between them, batch sizes that make later calls grow the context's scratch while earlier
    ones may still run, row updates on a fourth stream, an accumulating call, an expansion and a host evaluation
    in the chain; each result is the oracle's for the table as it stood when the call was enqueued;
  * test_one_context_handed_between_threads: threads take turns with one context under a lock, each enqueueing
    on its own stream and handing over without synchronising.

Oracles: tests/plan_matrix.py (plain contexts of up to 32 columns), tests/wide_oracle.py (wider, and where the
batches are large), the trimmed tables' oracle of tests/test_gpu_trimmed.py restated below, and per-bin
plan_matrix oracles for the grouped context.  Every worker is joined with a deadline: one that has not finished
fails the test with its name and the step it is at."""
import os
import sys
import threading
import time
import traceback

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402
import plan_matrix as PM  # noqa: E402
import wide_oracle as WO  # noqa: E402
import xor_oracle  # noqa: E402
from common import random_table  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

D, S, C, A = B.PRF_DUMMY, B.PRF_SALSA20, B.PRF_CHACHA20, B.PRF_AES128
SUFFIX = {"standard": "", "et": "_et", "xor": "_xor"}
ROUNDS = 20
DEADLINE = 150.0      # seconds for all threads of one test, from the first start


# ---- threads with a name, a current step and a deadline ---------------------------------------------------

class Worker(threading.Thread):
    """runs script(self) on its own thread; self.at() records the step it is at, self.ready() waits for the
    other workers to be set up"""

    def __init__(self, name, script):
        super().__init__(name=name, daemon=True)
        self.script, self.barrier = script, None
        self.step, self.error = "not started", None

    def at(self, step):
        self.step = step

    def ready(self):
        self.at("waiting for the other workers")
        self.barrier.wait()

    def run(self):
        try:
            self.script(self)
            self.step = "done"
        except threading.BrokenBarrierError:
            self.error = "the start barrier broke (another worker failed while setting up)"
        except BaseException:   # noqa: B902 -- reported by run_workers with the worker's name and step
            self.error = "at %s:\n%s" % (self.step, traceback.format_exc())
            if self.barrier is not None:
                self.barrier.abort()


def run_workers(workers, deadline=DEADLINE):
    barrier = threading.Barrier(len(workers), timeout=deadline)
    for w in workers:
        w.barrier = barrier
    end = time.monotonic() + deadline
    for w in workers:
        w.start()
    for w in workers:
        w.join(max(0.0, end - time.monotonic()))
    late = ["%s (at %s)" % (w.name, w.step) for w in workers if w.is_alive()]
    assert not late, "workers still running after %.0f s: %s" % (deadline, ", ".join(late))
    errors = ["%s failed %s" % (w.name, w.error) for w in workers if w.error is not None]
    broken = [e for e in errors if "start barrier broke" not in e]
    assert not errors, "\n".join(broken or errors)


def check(got, want, where):
    got = np.asarray(got)
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).reshape(len(want), -1).any(axis=1))[0] if got.shape == want.shape else []
        raise AssertionError("%s: result differs from the oracle (shape %s, want %s; rows %s)"
                             % (where, got.shape, want.shape, list(bad[:8])))


def accumulated(kind, base, res):
    b, r = base.view(np.uint32), res.view(np.uint32)
    return (b ^ r if kind == "xor" else b + r).view(np.int32)


def trimmed_expected(kind, prf, keys, table):
    """a trimmed table's oracle (tests/test_gpu_trimmed.py): row r is read at key index trimmed_alpha(r)"""
    n = table.shape[0]
    order = np.array([B.trimmed_alpha(r, n, SUFFIX[kind]) for r in range(n)], np.int64)
    keys = np.asarray(keys, np.int32).reshape(-1, 524)
    if kind == "xor":
        bits = np.stack([xor_oracle.unpack_bits(B.eval_cpu_xor(k, prf)) for k in keys])
        return xor_oracle.xor_rows(bits[:, order], table)
    ev = B.eval_cpu if kind == "standard" else B.eval_cpu_et
    return WO.dot_u32_exact(np.stack([ev(k, prf) for k in keys])[:, order], table)


def pick_rows(n, count, rng):
    rows = rng.randint(0, n, size=count).astype(np.int64)
    rows[:min(count, 2)] = [n - 1, 0][:min(count, 2)]
    return rows


def round_of(batches, r):
    """round r's batch size and server (0: keys a, 1: keys b): every batch size meets both servers"""
    return batches[r % len(batches)], (r // len(batches)) % 2


# ---- the workers of test_independent_contexts_on_threads: prepared on the main thread -----------------------

def plain_worker(name, kind, prf, n, e, batches, options=(), updates=False, trimmed=False, seed=0):
    """a Context of its own: every round through eval, eval_packed, eval_gather, eval_device on the worker's
    stream and eval_device(accumulate=True); with `updates`, update_rows after every round"""
    rng = np.random.RandomState(seed)
    table = random_table(n, e, seed=seed)
    sfx = SUFFIX[kind]
    keys = {}
    for b in sorted(set(batches)):
        rows = pick_rows(n, b, rng)
        idx = np.array([B.trimmed_alpha(int(r), n, sfx) for r in rows], np.int64) if trimmed else rows
        ka, kb = PM.gen_keys(kind, B.trimmed_domain(n, sfx) if trimmed else n, idx, prf, seed=seed + b)
        keys[b] = (rows, (ka, kb))
    versions, upd = [table], []
    if updates:
        for r in range(ROUNDS):
            idx = rng.randint(0, n, size=3).astype(np.int64)
            idx[2] = idx[0]                                  # a duplicate: the last occurrence wins
            new = random_table(3, e, seed=seed * 1000 + r)
            t = versions[-1].copy()
            for j in range(3):
                t[idx[j]] = new[j]
            upd.append((idx, new))
            versions.append(t)
    if trimmed:
        oracle = trimmed_expected
    else:
        oracle = PM.expected if e <= 32 else WO.expected
    cache = {}

    def want_of(b, side, v):
        if (b, side, v) not in cache:
            cache[b, side, v] = oracle(kind, prf, keys[b][1][side], versions[v])
        return cache[b, side, v]
    for b in keys:         # both servers' results reconstruct the selected rows
        rows = keys[b][0]
        assert np.array_equal(PM.reconstruct(kind, want_of(b, 0, 0), want_of(b, 1, 0)), table[rows]), (name, b)
    wants = [want_of(*round_of(batches, r), r if updates else 0) for r in range(ROUNDS)]

    pack = getattr(B, "key_pack" + sfx)
    packed = {(b, s): b"".join(pack(k) for k in keys[b][1][s]) for b in keys for s in (0, 1)}
    keys_dev = {(b, s): torch.from_numpy(keys[b][1][s]).cuda() for b in keys for s in (0, 1)}
    base = {b: random_table(b, e, seed=seed + 7 * b) for b in keys}
    base_dev = {b: torch.from_numpy(base[b]).cuda() for b in keys}
    out = {b: torch.empty((b, e), dtype=torch.int32, device="cuda") for b in keys}
    acc = {b: torch.empty((b, e), dtype=torch.int32, device="cuda") for b in keys}

    def script(w):
        w.at("create")
        ctx = B.Context(table, early_termination=kind == "et", xor=kind == "xor", trimmed=trimmed)
        try:
            for opt, value in options:
                ctx.set_option(opt, value)
            stream = torch.cuda.Stream()
            w.ready()
            for r in range(ROUNDS):
                b, side = round_of(batches, r)
                k, want = keys[b][1][side], wants[r]
                where = "%s round %d (%d keys, server %s)" % (name, r, b, "ab"[side])
                w.at(where + " eval")
                check(ctx.eval(k, prf), want, where + " eval")
                w.at(where + " eval_packed")
                check(ctx.eval_packed(packed[b, side], b, prf), want, where + " eval_packed")
                w.at(where + " eval_gather")
                check(ctx.eval_gather(list(k), prf), want, where + " eval_gather")
                w.at(where + " eval_device")
                with torch.cuda.stream(stream):
                    out[b].fill_(-1)
                    ctx.eval_device(keys_dev[b, side].data_ptr(), b, prf, out[b].data_ptr(), stream=stream.cuda_stream)
                    acc[b].copy_(base_dev[b])
                    ctx.eval_device(keys_dev[b, side].data_ptr(), b, prf, acc[b].data_ptr(), stream=stream.cuda_stream,
                                    accumulate=True)
                stream.synchronize()
                check(out[b].cpu().numpy(), want, where + " eval_device")
                check(acc[b].cpu().numpy(), accumulated(kind, base[b], want), where + " eval_device(accumulate)")
                if updates:
                    w.at(where + " update_rows")
                    ctx.update_rows(*upd[r])
        finally:
            ctx.close()
    return Worker(name, script)


def grouped_worker(name, kind, prf, sizes, e, nqs, seed=0):
    """a GroupContext of its own: every round through eval, eval_device and eval_queries_device (wire and
    compact) on the worker's stream, each checked against per-bin oracles"""
    rng = np.random.RandomState(seed)
    tables = [random_table(m, e, seed=seed + g) for g, m in enumerate(sizes)]
    nbins = len(sizes)
    q = {}
    for nq in sorted(set(nqs)):
        rows = np.stack([pick_rows(m, nq, rng) for m in sizes], axis=1)
        ka = np.zeros((nq, nbins, 524), np.int32)
        kb = np.zeros_like(ka)
        for g, m in enumerate(sizes):
            ka[:, g], kb[:, g] = PM.gen_keys(kind, m, rows[:, g], prf, seed=seed + 31 * nq + g)
        want = []
        for keys in (ka, kb):
            w = np.zeros((nq, nbins, e), np.int32)
            for g in range(nbins):
                w[:, g] = PM.expected(kind, prf, keys[:, g], tables[g])
            want.append(w)
        for g in range(nbins):
            assert np.array_equal(PM.reconstruct(kind, want[0][:, g], want[1][:, g]), tables[g][rows[:, g]]), (name, g)
        q[nq] = ((ka, kb), want)
    bins = {nq: np.tile(np.arange(nbins, dtype=np.int32), nq) for nq in q}
    perm = {nq: np.random.RandomState(nq).permutation(nq * nbins) for nq in q}
    dev = {}
    for nq, ((ka, kb), _) in q.items():
        for s, keys in enumerate((ka, kb)):
            flat = keys.reshape(-1, 524)
            dev[nq, s] = (torch.from_numpy(keys).cuda(), torch.from_numpy(np.ascontiguousarray(flat[perm[nq]])).cuda())
    outs = {nq: torch.empty((nq, nbins, e), dtype=torch.int32, device="cuda") for nq in q}
    flat_outs = {nq: torch.empty((nq * nbins, e), dtype=torch.int32, device="cuda") for nq in q}

    def script(w):
        w.at("create")
        ctx = B.GroupContext(tables, early_termination=kind == "et", xor=kind == "xor")
        try:
            compact = {(nq, s): torch.from_numpy(ctx.pack_queries(q[nq][0][s])).cuda() for nq in q for s in (0, 1)}
            stream = torch.cuda.Stream()
            torch.cuda.synchronize()
            w.ready()
            for r in range(ROUNDS):
                nq, side = round_of(nqs, r)
                keys, want = q[nq][0][side], q[nq][1][side]
                where = "%s round %d (%d queries, server %s)" % (name, r, nq, "ab"[side])
                w.at(where + " eval")
                check(ctx.eval(keys.reshape(-1, 524), bins[nq], prf).reshape(want.shape), want, where + " eval")
                w.at(where + " eval_device")
                wire, shuffled = dev[nq, side]
                with torch.cuda.stream(stream):
                    flat_outs[nq].fill_(-1)
                    ctx.eval_device(shuffled.data_ptr(), bins[nq][perm[nq]], prf, flat_outs[nq].data_ptr(),
                                    stream=stream.cuda_stream)
                stream.synchronize()
                check(flat_outs[nq].cpu().numpy(), want.reshape(-1, e)[perm[nq]], where + " eval_device")
                for fmt, src in (("wire", wire), ("compact", compact[nq, side])):
                    w.at(where + " eval_queries_device " + fmt)
                    with torch.cuda.stream(stream):
                        outs[nq].fill_(-1)
                        ctx.eval_queries_device(src.data_ptr(), nq, prf, outs[nq].data_ptr(), stream=stream.cuda_stream,
                                                compact=fmt == "compact")
                    stream.synchronize()
                    check(outs[nq].cpu().numpy(), want, where + " eval_queries_device " + fmt)
        finally:
            ctx.close()
    return Worker(name, script)


def dpf_worker(name, prf, n, e, batches, seed=0):
    """a dpf.DPF object (the pybind binding, which releases the GIL around its calls): eval_gpu from a key
    tensor and from a key list, eval_gpu_compact, eval_gpu_device on the worker's stream and accumulating"""
    import dpf
    rng = np.random.RandomState(seed)
    table = random_table(n, e, seed=seed)
    keys, wants = {}, {}
    for b in sorted(set(batches)):
        rows = pick_rows(n, b, rng)
        ka, kb = PM.gen_keys("standard", n, rows, prf, seed=seed + b)
        wa, wb = PM.expected("standard", prf, ka, table), PM.expected("standard", prf, kb, table)
        assert np.array_equal(PM.reconstruct("standard", wa, wb), table[rows]), (name, b)
        keys[b], wants[b] = (ka, kb), (wa, wb)
    keys_dev = {(b, s): torch.from_numpy(keys[b][s]).cuda() for b in keys for s in (0, 1)}
    base = {b: random_table(b, e, seed=seed + 3 * b) for b in keys}
    base_dev = {b: torch.from_numpy(base[b]).cuda() for b in keys}
    acc = {b: torch.empty((b, e), dtype=torch.int32, device="cuda") for b in keys}

    def script(w):
        w.at("create")
        d = dpf.DPF(prf=prf)
        try:
            d.eval_init(torch.from_numpy(table))
            stream = torch.cuda.Stream()
            w.ready()
            for r in range(ROUNDS):
                b, side = round_of(batches, r)
                k, want = torch.from_numpy(keys[b][side]), wants[b][side]
                where = "%s round %d (%d keys, server %s)" % (name, r, b, "ab"[side])
                w.at(where + " eval_gpu")
                check(d.eval_gpu(k).numpy(), want, where + " eval_gpu")
                w.at(where + " eval_gpu(list)")
                check(d.eval_gpu(list(k)).numpy(), want, where + " eval_gpu(list)")
                w.at(where + " eval_gpu_compact")
                check(d.eval_gpu_compact(d.pack_keys(k)).numpy(), want, where + " eval_gpu_compact")
                w.at(where + " eval_gpu_device")
                with torch.cuda.stream(stream):
                    out = d.eval_gpu_device(keys_dev[b, side])
                    acc[b].copy_(base_dev[b])
                    d.eval_gpu_device(keys_dev[b, side], out_dev=acc[b], accumulate=True)
                stream.synchronize()
                check(out.cpu().numpy(), want, where + " eval_gpu_device")
                check(acc[b].cpu().numpy(), accumulated("standard", base[b], want), where + " eval_gpu_device(accumulate)")
        finally:
            d.close()
    return Worker(name, script)


def keygen_worker(name, rounds=6, seed=0):
    """b200dpf_gen_batch_gpu, _et and _xor, each against the host generator's keys for the same seeds"""
    rng = np.random.RandomState(seed)
    jobs = []
    for r in range(rounds):
        for kind, n in (("standard", 1 << 12), ("et", 1 << 12), ("xor", 1 << 14)):
            alphas = pick_rows(n, 40, rng)
            seeds = rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()
            prf = (r + len(jobs)) % 4
            cpu = {"standard": B.gen_batch_secure, "et": B.gen_batch_et, "xor": B.gen_batch_xor}[kind]
            jobs.append((kind, n, prf, alphas, seeds, cpu(alphas, n, seeds, prf)))

    def script(w):
        w.ready()
        for i, (kind, n, prf, alphas, seeds, (ha, hb)) in enumerate(jobs):
            where = "%s job %d (%s keys, %s)" % (name, i, kind, B.PRF_NAMES[prf])
            w.at(where)
            ga, gb = getattr(B, "gen_batch_gpu" + SUFFIX[kind])(alphas, n, seeds, prf)
            check(ga, ha, where + " key a")
            check(gb, hb, where + " key b")
    return Worker(name, script)


def churn_worker(name, iterations=12, seed=0):
    """creates a context, evaluates once, checks and destroys it, over and over while the others run: creation
    probes the shared-memory base and writes the AES constant table"""
    jobs = []
    for prf, n, e in ((C, 1 << 11, 16), (A, 1 << 10, 8), (S, 1 << 9, 20)):
        table = random_table(n, e, seed=seed + n)
        rows = pick_rows(n, 16, np.random.RandomState(n))
        ka, _ = PM.gen_keys("standard", n, rows, prf, seed=seed + prf)
        jobs.append((prf, table, ka, PM.expected("standard", prf, ka, table)))

    def script(w):
        w.ready()
        for i in range(iterations):
            prf, table, ka, want = jobs[i % len(jobs)]
            where = "%s iteration %d (%s, n=%d)" % (name, i, B.PRF_NAMES[prf], table.shape[0])
            w.at(where + " create")
            ctx = B.Context(table)
            try:
                w.at(where + " eval")
                check(ctx.eval(ka, prf), want, where)
                w.at(where + " destroy")
            finally:
                ctx.close()
    return Worker(name, script)


# The three ChaCha20 workers launch one kernel, dpf_eval_kernel<ChaCha20, 4, MODE_FUSED> (standard keys,
# 16 columns, 256 threads: level_bytes = 4096), each with its own dynamic shared memory.  With the frontier off
# there is no tree-top stack, so (dpf_plan.cu smem_layout / smem_bytes)
#     smem = off_lo + (s - 1) * 4096,   off_lo = 2048 * depth + 1040   (correction words, level-0 words, roots)
# and s is subtree_log2 (below depth and s_max):
#     n = 2^10, s = 2:  20480 + 1040 +  4096 = 25616 bytes
#     n = 2^12, s = 4:  24576 + 1040 + 12288 = 37904 bytes
#     n = 2^14, s = 6:  28672 + 1040 + 20480 = 50192 bytes
# The 160-column worker's leaf-caching pass and the churn worker's n = 2^11 context run that kernel too, at
# sizes the automatic work-item choice gives.
CHACHA_SIZES = ((1 << 10, 2), (1 << 12, 4), (1 << 14, 6))


def independent_workers():
    (n0, s0), (n1, s1), (n2, s2) = CHACHA_SIZES
    return [
        plain_worker("chacha-n2^10", "standard", C, n0, 16, (1, 5, 33, 64, 3),
                     options=(("frontier", 0), ("subtree_log2", s0)), seed=1),
        plain_worker("chacha-n2^12", "standard", C, n1, 16, (40, 2, 17, 100, 7),
                     options=(("frontier", 0), ("subtree_log2", s1)), updates=True, seed=2),
        plain_worker("chacha-n2^14", "standard", C, n2, 16, (64, 9, 1, 32, 200),
                     options=(("frontier", 0), ("subtree_log2", s2)), seed=3),
        plain_worker("et-aes", "et", A, 1 << 12, 20, (3, 33, 1, 64, 20), updates=True, seed=4),
        plain_worker("xor-salsa", "xor", S, 1 << 14, 16, (1, 4, 33, 128, 6), seed=5),
        plain_worker("trimmed-et-dummy", "et", D, 3001, 20, (2, 40, 1, 17, 5), updates=True, trimmed=True, seed=6),
        plain_worker("wide-chacha-E160", "standard", C, 1 << 12, 160, (17, 64, 5, 100, 33),
                     options=(("leaf_cache_mb", 1),), seed=7),
        grouped_worker("grouped-salsa", "standard", S, (2, 64, 1 << 10, 1 << 12), 16, (1, 3, 8, 2, 5), seed=8),
        dpf_worker("dpf-object-aes", A, 1 << 11, 24, (1, 16, 48, 7, 3), seed=9),
        keygen_worker("keygen-gpu", seed=10),
        churn_worker("create-destroy", seed=11),
    ]


def test_independent_contexts_on_threads():
    B.lib()
    import dpf  # noqa: F401  (the binding loads here, before any thread starts)
    workers = independent_workers()
    torch.cuda.synchronize()
    run_workers(workers)


# ---- one context, many streams ------------------------------------------------------------------------------

# (batch, stream): streams 0..2 rotate; the batch sizes move the lane split, the keys per warp, the work-item
# size and the frontier, and the 512- and 2000-key calls grow the counters, the frontier and the leaf cache
# while the calls before them may still run
CHAIN = [(1, 0), (5, 1), (33, 2), (512, 0), "update", (2000, 1), "accumulate", "expand", "host", (1000, 2),
         (17, 0), (2, 1), (300, 2), (700, 0)]
STREAM_CASES = [(kind, prf, e) for kind in PM.KINDS for prf, e in ((C, 16), (A, 16), (S, 160))]


@pytest.mark.parametrize("kind,prf,e", STREAM_CASES,
                         ids=["%s-%s-E%d" % (k, B.PRF_NAMES[p], e) for k, p, e in STREAM_CASES])
def test_one_context_many_streams(kind, prf, e):
    n = 1 << 12
    rng = np.random.RandomState(e + prf)
    table = random_table(n, e, seed=e + prf)
    rows = pick_rows(n, 2000, rng)
    ka, kb = PM.gen_keys(kind, n, rows, prf, seed=e)
    upd_idx = rng.randint(0, n, size=9).astype(np.int64)
    upd_idx[:3] = [rows[0], rows[4], rows[1]]             # rows the keys select
    upd_rows = random_table(len(upd_idx), e, seed=e + 1)
    updated = table.copy()
    for j, i in enumerate(upd_idx):
        updated[i] = upd_rows[j]
    # the oracle of both table versions for the whole key pool (each call takes a prefix of it)
    before, after = WO.expected(kind, prf, ka, table), WO.expected(kind, prf, ka, updated)
    b_before, b_after = WO.expected(kind, prf, kb[:64], table), WO.expected(kind, prf, kb[:64], updated)
    assert np.array_equal(PM.reconstruct(kind, before[:64], b_before), table[rows[:64]])
    assert np.array_equal(PM.reconstruct(kind, after[:64], b_after), updated[rows[:64]])
    shares = PM.expected_shares(kind, prf, ka[:3])

    ctx = B.Context(table, early_termination=kind == "et", xor=kind == "xor")
    if e > 16:
        ctx.set_option("leaf_cache_mb", 1)          # leaf-cache chunks of a few key groups
    streams = [torch.cuda.Stream() for _ in range(4)]
    keys_a, keys_b = torch.from_numpy(ka).cuda(), torch.from_numpy(kb[:64]).cuda()
    i_dev, r_dev = torch.from_numpy(upd_idx).cuda(), torch.from_numpy(upd_rows).cuda()
    acc = torch.full((5, e), -1, dtype=torch.int32, device="cuda")
    width = n // 32 if kind == "xor" else n
    expand_out = torch.full((3, width), -1, dtype=torch.int32, device="cuda")
    outs = {step: torch.full((step[0], e), -1, dtype=torch.int32, device="cuda") for step in CHAIN if isinstance(step, tuple)}
    checks, host = [], None
    torch.cuda.synchronize()          # from here on, nothing waits on the host until the end
    try:
        updated_yet = False
        for step in CHAIN:
            if step == "update":
                ctx.update_rows_device(i_dev.data_ptr(), r_dev.data_ptr(), len(upd_idx), stream=streams[3].cuda_stream)
                updated_yet = True
            elif step == "accumulate":   # into a buffer an earlier call of the chain filled, on another stream
                ctx.eval_device(keys_b.data_ptr(), 5, prf, acc.data_ptr(), stream=streams[2].cuda_stream)
                ctx.eval_device(keys_a.data_ptr(), 5, prf, acc.data_ptr(), stream=streams[0].cuda_stream, accumulate=True)
                checks.append(("accumulate", acc, accumulated(kind, b_after[:5], after[:5])))
            elif step == "expand":
                ctx.expand_device(keys_a.data_ptr(), 3, prf, expand_out.data_ptr(), stream=streams[1].cuda_stream)
                checks.append(("expand_device", expand_out, shares))
            elif step == "host":
                host = ctx.eval(kb[:64], prf)
            else:
                batch, s = step
                ctx.eval_device(keys_a.data_ptr(), batch, prf, outs[step].data_ptr(), stream=streams[s].cuda_stream)
                checks.append(("%d keys on stream %d" % step, outs[step], (after if updated_yet else before)[:batch]))
        torch.cuda.synchronize()
    finally:
        ctx.close()
    where = "%s-%s-E%d" % (kind, B.PRF_NAMES[prf], e)
    check(host, b_after, where + " host eval in the chain")
    for what, got, want in checks:
        got = got.cpu().numpy()
        check(got.view(np.uint32) if what == "expand_device" and kind == "xor" else got, want, where + " " + what)


# ---- one context handed between threads ---------------------------------------------------------------------

@pytest.mark.parametrize("prf", [C, A], ids=lambda p: B.PRF_NAMES[p])
def test_one_context_handed_between_threads(prf):
    """threads take turns with one context under a lock (one host thread at a time); each enqueues eval_device
    on its own stream and hands over without synchronising, so the next thread's call (another batch size, often
    a larger scratch) is ordered behind work that may still run"""
    n, e, threads, turns = 1 << 12, 16, 4, 5
    batches = (1, 700, 3, 64, 2000, 17, 250, 5, 1200, 40)
    table = random_table(n, e, seed=prf)
    rows = pick_rows(n, max(batches), np.random.RandomState(prf))
    ka, kb = PM.gen_keys("standard", n, rows, prf, seed=prf)
    want = WO.expected("standard", prf, ka, table)
    assert np.array_equal(PM.reconstruct("standard", want[:40], WO.expected("standard", prf, kb[:40], table)), table[rows[:40]])
    keys_dev = torch.from_numpy(ka).cuda()
    outs = [[torch.full((batches[(t * turns + i) % len(batches)], e), -1, dtype=torch.int32, device="cuda")
             for i in range(turns)] for t in range(threads)]
    ctx = B.Context(table)
    lock = threading.Lock()
    torch.cuda.synchronize()

    def turn_script(t):
        def script(w):
            stream = torch.cuda.Stream()
            w.ready()
            for i in range(turns):
                out = outs[t][i]
                w.at("turn %d (%d keys)" % (i, out.shape[0]))
                with lock:
                    ctx.eval_device(keys_dev.data_ptr(), out.shape[0], prf, out.data_ptr(), stream=stream.cuda_stream)
        return script
    try:
        run_workers([Worker("thread-%d" % t, turn_script(t)) for t in range(threads)])
        torch.cuda.synchronize()
    finally:
        ctx.close()
    for t in range(threads):
        for i, out in enumerate(outs[t]):
            check(out.cpu().numpy(), want[:out.shape[0]], "thread %d turn %d (%d keys)" % (t, i, out.shape[0]))
