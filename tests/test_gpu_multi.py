"""Entry-range sharding across real GPUs: one process per GPU with an NCCL reduce of the partials
(ShardedDPF), and one process driving every GPU (b200dpf_create_multi, peer-memory reduction).
The multi-device tests need >= 2 CUDA devices (skipped on a 1-GPU box); the single-process
context with a one-device list runs anywhere."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    for sub in ("gpu-dpf_b200", "oracle", "tests"):
        sys.path.insert(0, os.path.join(ROOT, sub))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import b200dpf
    import oracle as O
    from common import random_table, seeded_keys
    from sharded import ShardedDPF
    orc = O.Oracle()
    n = 1 << 14
    table = random_table(n, 16, seed=13)
    for prf, axis, reduce in ((3, "entries", "nccl"), (2, "entries", "nccl"), (3, "entries", "fused"),
                              (1, "entries", "fused"), (3, "keys", "nccl")):
        ka, kb, idx = seeded_keys(b200dpf.gen, n, 70, prf, seed=17)
        d = ShardedDPF(prf=prf, axis=axis, reduce=reduce)
        d.eval_init(torch.from_numpy(table))
        got_a = d.eval_gpu(torch.from_numpy(ka))
        got_b = d.eval_gpu([torch.from_numpy(k) for k in kb])
        if rank == 0:
            assert np.array_equal(got_a.numpy()[:8], orc.eval_dot(ka[:8], prf, table))
            rec = (got_a.numpy().astype(np.uint32) - got_b.numpy().astype(np.uint32)).astype(np.int32)
            assert np.array_equal(rec, table[idx])
        else:
            assert got_a is None
        d.close()
    # BASELINE config 5 shape (scaled down): entry_size 128, AES128, sharded, batch not a multiple of 32
    n, entry, prf = 1 << 16, 128, 3
    table = random_table(n, entry, seed=5)
    ka, kb, idx = seeded_keys(b200dpf.gen, n, 45, prf, seed=6)
    d = ShardedDPF(prf=prf)
    d.eval_init(torch.from_numpy(table))
    got_a, got_b = d.eval_gpu(torch.from_numpy(ka)), d.eval_gpu(torch.from_numpy(kb))
    if rank == 0:
        rec = (got_a.numpy().astype(np.uint32) - got_b.numpy().astype(np.uint32)).astype(np.int32)
        assert np.array_equal(rec, table[idx])
        assert np.array_equal(got_a.numpy()[:2], orc.eval_dot(ka[:2], prf, table))
    d.close()
    if rank == 0:
        ret.put("ok")
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_nccl():
    world = torch.cuda.device_count()
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 1 << (world.bit_length() - 1)
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, ret)) for r in range(world)]
    [p.start() for p in procs]
    [p.join(300) for p in procs]
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert ret.get(timeout=5) == "ok"


def _devices():
    n = torch.cuda.device_count()
    return list(range(1 << (n.bit_length() - 1))) if n else []


def test_multi_context_with_one_device():
    """b200dpf_create_multi degenerates cleanly: one device, either axis, same results as a plain context."""
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    for sub in ("gpu-dpf_b200", "oracle", "tests"):
        sys.path.insert(0, os.path.join(ROOT, sub))
    import b200dpf
    import oracle as O
    from common import random_table, seeded_keys
    n, prf = 4096, 3
    table = random_table(n, 16, seed=71)
    ka, _, _ = seeded_keys(b200dpf.gen, n, 70, prf, seed=72)
    want = O.Oracle().eval_dot(ka, prf, table)
    for axis in (0, 1, 2):
        ctx = b200dpf.Context.multi(table, [0], axis)
        assert ctx.device_count == 1
        assert np.array_equal(ctx.eval(ka, prf), want)
        packed = b"".join(b200dpf.key_pack(k) for k in ka)
        assert np.array_equal(ctx.eval_packed(packed, 70, prf), want)
        ctx.close()


def test_single_process_all_gpus():
    """One process, every GPU of the box behind ONE context: entry-range shards with the
    peer-memory reduction, key-split replicas, and the automatic choice."""
    devs = _devices()
    if len(devs) < 2:
        pytest.skip("needs >= 2 GPUs")
    for sub in ("gpu-dpf_b200", "oracle", "tests"):
        sys.path.insert(0, os.path.join(ROOT, sub))
    import b200dpf
    import oracle as O
    from common import oracle_dot_mt, random_table, seeded_keys
    orc = O.Oracle()
    for n, entry, batch, prf in ((1 << 14, 16, 70, 3), (1 << 14, 16, 600, 1), (1 << 19, 16, 513, 2), (1 << 16, 128, 45, 3),
                                 (1 << 12, 5, 3, 0)):
        table = random_table(n, entry, seed=n + entry)
        ka, kb, idx = seeded_keys(b200dpf.gen, n, batch, prf, seed=batch)
        want = oracle_dot_mt(orc, ka[:8], prf, table)
        for axis in (1, 2, 0):
            ctx = b200dpf.Context.multi(table, devs, axis)
            assert ctx.device_count == len(devs)
            assert ctx.axis == (axis if axis else (2 if n <= (1 << 18) else 1))
            a, b = ctx.eval(ka, prf), ctx.eval(kb, prf)
            assert np.array_equal(a[:8], want), (n, entry, batch, prf, axis)
            assert np.array_equal((a.astype(np.uint32) - b.astype(np.uint32)).astype(np.int32), table[idx])
            packed = b"".join(b200dpf.key_pack(k) for k in ka)
            assert np.array_equal(ctx.eval_packed(packed, batch, prf), a)
            for _ in range(3):                    # back-to-back calls reuse the worker threads
                assert np.array_equal(ctx.eval(ka, prf), a)
            ctx.close()


def test_python_api_devices_all():
    """dpf.DPF(devices='all'), and the B200DPF_DEVICES switch that lets callers of the reference's
    pybind interface (eval_init(table) has no device argument) use every GPU."""
    devs = _devices()
    if len(devs) < 2:
        pytest.skip("needs >= 2 GPUs")
    for sub in ("gpu-dpf_b200", "oracle", "tests"):
        sys.path.insert(0, os.path.join(ROOT, sub))
    import subprocess
    import dpf
    import dpf_cpp
    from common import random_table
    n = 1 << 15
    table = torch.from_numpy(random_table(n, 16, seed=5))
    d = dpf.DPF(prf=dpf.DPF.PRF_SALSA20, devices="all", axis="entries")
    d.eval_init(table)
    assert dpf_cpp.device_count(d.buffers) == torch.cuda.device_count() and dpf_cpp.axis(d.buffers) == 1
    idx = [0, 777, n - 1]
    keys = [d.gen(i, n) for i in idx]
    a = d.eval_gpu([k[0] for k in keys])
    b = d.eval_gpu(torch.stack([k[1] for k in keys]))
    assert torch.equal(a - b, table[idx])
    d.close()
    # the reference's calling convention (sample.py's query: entry 42 of a 2^14-row table, a batch of
    # exactly 512 keys) in a fresh process whose environment asks for every GPU
    script = (
        "import torch, dpf_cpp\n"
        "n = 16384\n"
        "table = torch.randint(2**31, (n, 16), generator=torch.Generator().manual_seed(5)).int()\n"
        "table[42] = 42\n"
        "k1, k2 = dpf_cpp.gen(42, n, bytes(128), dpf_cpp.PRF_AES128)\n"
        "buf = dpf_cpp.eval_init(table)\n"
        "assert dpf_cpp.device_count(buf) == torch.cuda.device_count(), dpf_cpp.device_count(buf)\n"
        "r = dpf_cpp.eval_gpu([k1, k2] + [k2] * 510, buf, n, dpf_cpp.PRF_AES128).cpu()\n"
        "assert tuple(r.shape) == (512, 16) and torch.equal(r[0] - r[1], table[42]), r[:2]\n"
        "dpf_cpp.eval_free(buf)\n"
        "print('ok')\n")
    env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "gpu-dpf_b200"), B200DPF_DEVICES="all")
    r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
