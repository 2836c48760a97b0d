"""The host entry points on several threads at once (include/b200dpf.h, "Threading"): the last error message is
per thread, and key generation, host evaluation, trimmed key indices and the compact key form give the same
bytes on 8 threads at once as on one.  ctypes releases the GIL around every call, so the threads really do run
the library at the same time."""
import os
import sys
import threading
import traceback

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "gpu-dpf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import b200dpf as B  # noqa: E402

THREADS = 8
DEADLINE = 120.0     # seconds for every thread of one test to finish


def run_threads(work, count=THREADS):
    """work(t) on `count` threads started together; the first failure (with its thread) is raised, and a thread
    still running at the deadline fails the test instead of hanging it"""
    errors = [None] * count

    def body(t):
        try:
            work(t)
        except BaseException:   # noqa: B902 -- reported below, with the thread's number
            errors[t] = traceback.format_exc()
    threads = [threading.Thread(target=body, args=(t,), name="host-%d" % t, daemon=True) for t in range(count)]
    for th in threads:
        th.start()
    for th in threads:
        th.join(DEADLINE)
    late = [th.name for th in threads if th.is_alive()]
    assert not late, "threads still running after %.0f s: %s" % (DEADLINE, late)
    for t, err in enumerate(errors):
        assert err is None, "thread %d failed:\n%s" % (t, err)


def test_last_error_is_per_thread():
    """Each thread makes its own failing call, all threads wait until every call has failed, then each reads
    b200dpf_last_error: it must be its own call's message, not the last one made in the process."""
    L = B.lib()
    rounds = 4
    barrier = threading.Barrier(THREADS, timeout=DEADLINE)
    key = B.gen_batch_secure(np.array([3], np.int64), 64, bytes(44), B.PRF_DUMMY)[0][0]
    out = np.zeros(64, np.int32)

    def work(t):
        for r in range(rounds):
            if t % 2 == 0:
                got = 1 + t + THREADS * r            # a seed too short by a length of this thread's own
                rc = L.b200dpf_gen_secure(3, 64, bytes(got), got, B.PRF_DUMMY, np.zeros(B.KEY_WORDS, np.int32),
                                          np.zeros(B.KEY_WORDS, np.int32))
                want = "needs at least 44 bytes of seed (got %d)" % got
            else:
                prf = 100 + t + THREADS * r          # a PRF id of this thread's own
                rc = L.b200dpf_eval_cpu(key, prf, out)
                want = "unknown prf id %d" % prf
            assert rc != 0, (t, r)
            barrier.wait()                          # every thread's call has failed
            msg = L.b200dpf_last_error().decode()
            assert want in msg, "thread %d round %d read %r, its own call said %r" % (t, r, msg, want)
            barrier.wait()                          # every thread has read before the next round fails again
    run_threads(work)


def _kinds():
    return (("", B.gen_batch_secure, B.eval_cpu, B.key_pack, B.key_unpack),
            ("_et", B.gen_batch_et, B.eval_cpu_et, B.key_pack_et, B.key_unpack_et),
            ("_xor", B.gen_batch_xor, B.eval_cpu_xor, B.key_pack_xor, B.key_unpack_xor))


def _job(j):
    """job j: (kind suffix, n, prf, alphas, seed bytes), with every kind and PRF among the jobs"""
    rng = np.random.RandomState(j)
    kind = ("", "_et", "_xor")[j % 3]
    n = {"": 1 << (4 + j % 7), "_et": 1 << (5 + j % 6), "_xor": 1 << (8 + j % 5)}[kind]
    alphas = rng.randint(0, n, size=1 + j % 5).astype(np.int64)
    alphas[0] = n - 1
    return kind, n, (j // 3) % 4, alphas, rng.randint(0, 256, size=44 * len(alphas)).astype(np.uint8).tobytes()


def _compute(j):
    """everything job j makes on the host: both keys of every alpha (DRBG and 32-bit seeds), their host
    evaluations, their compact forms and those unpacked again, and trimmed key indices"""
    kind, n, prf, alphas, seeds = _job(j)
    gen, ev, pack, unpack = {k[0]: k[1:] for k in _kinds()}[kind]
    a, b = gen(alphas, n, seeds, prf, nthreads=1 + j % 3)
    res = [a, b]
    if kind == "":
        res += list(B.gen_batch(alphas, n, np.arange(len(alphas)) + 7 * j, prf, nthreads=1 + j % 2))
    for k in np.concatenate([a, b]):
        res.append(ev(k, prf))
        packed = pack(k)
        res.append(np.frombuffer(packed, np.uint8))
        res.append(unpack(packed))
    m = 1 + (j * 7919) % 5000
    res.append(np.array([B.trimmed_domain(m, kind)] + [B.trimmed_alpha(r, m, kind) for r in (0, m // 2, m - 1)],
                        np.int64))
    return res


def test_host_calls_match_one_thread():
    jobs = 48
    want = [_compute(j) for j in range(jobs)]
    got = [None] * jobs
    barrier = threading.Barrier(THREADS, timeout=DEADLINE)

    def work(t):
        barrier.wait()
        for j in range(t, jobs, THREADS):
            got[j] = _compute(j)
    run_threads(work)
    for j in range(jobs):
        assert len(got[j]) == len(want[j]), j
        for i, (g, w) in enumerate(zip(got[j], want[j])):
            assert np.array_equal(g, w), "job %d %s, result %d differs on 8 threads" % (j, _job(j)[:3], i)


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-q"]))
