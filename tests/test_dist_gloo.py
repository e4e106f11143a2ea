"""world_size-2 (and 3) CPU runs of the multi-GPU host logic over the gloo backend: sharding,
all-gather of partial results, folding.  The per-rank MSM is the CPU oracle here (there is no GPU
in this tier); on a GPU machine the same `parallel.msm_sharded` drives `sppark_b200_msm_dev` and
`sppark_b200_msm_combine` (bench.py --gpus N)."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, n, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from oracle import pyoracle as o
    from sppark_b200 import parallel
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    rng = np.random.default_rng(5)                       # same inputs on every rank
    pts = o.gen_points("bls12_381", 16)[np.arange(n) % 16].copy()
    sc = rng.integers(0, 2**63, size=(n, 4), dtype=np.uint64)
    sc[:, 3] >>= np.uint64(2)
    lo, hi = parallel.shard_range(n, rank, world)

    def local():
        return o.msm("bls12_381", pts[lo:hi], sc[lo:hi], "serial")

    def combine(parts):                                   # oracle stand-in for sppark_b200_msm_combine
        aff = np.stack([o.jac_to_affine("bls12_381", p) for p in parts])
        one = np.tile(np.array([1, 0, 0, 0], dtype=np.uint64), (len(parts), 1))
        return o.msm("bls12_381", aff, one, "naive")

    got = parallel.msm_sharded(local, combine, 18)
    want = o.msm("bls12_381", pts, sc, "serial")
    ok = np.array_equal(o.jac_to_affine("bls12_381", got), o.jac_to_affine("bls12_381", want))
    q.put((rank, bool(ok), (lo, hi)))
    dist.destroy_process_group()


@pytest.mark.parametrize("world,n", [(2, 101), (3, 64), (2, 1)])
def test_sharded_msm_over_gloo(world, n):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _ in res)
    ranges = sorted(r for _, _, r in res)
    assert ranges[0][0] == 0 and ranges[-1][1] == n
    assert all(ranges[i][1] == ranges[i + 1][0] for i in range(world - 1))


def test_shard_range_properties():
    sys.path.insert(0, ROOT)
    from sppark_b200 import parallel
    for n in (0, 1, 7, 64, 1 << 26):
        for world in (1, 2, 3, 8):
            r = [parallel.shard_range(n, g, world) for g in range(world)]
            assert r[0][0] == 0 and r[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(r, r[1:]))
            assert max(h - l for l, h in r) - min(h - l for l, h in r) <= 1


def _ntt_worker(rank, world, port, lg, q, split=None):
    sys.path.insert(0, ROOT)
    if split:
        os.environ["SPPARK_B200_NTT_SPLIT"] = split          # small digits: the multi-pass second stage
    s1 = int(split.split(",")[0]) if split else None
    import ctypes as C
    import torch
    import torch.distributed as dist
    from oracle import pyoracle as o
    from sppark_b200 import parallel
    emu = C.CDLL(os.path.join(ROOT, "tests", "emu", "libntt_emu.so"))
    emu.emu_ntt_slab_gl64.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint, C.c_uint, C.c_uint, C.c_int, C.c_uint]
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    lg_g = world.bit_length() - 1
    rng = np.random.default_rng(77)                      # same full input on every rank
    x = rng.integers(0, 2**64 - 2**32 + 1, size=1 << lg, dtype=np.uint64)
    local = torch.from_numpy(parallel.scatter_columns(x, lg, lg_g, rank, s1=s1).reshape(-1).view(np.int64).copy())

    def pass_fn(which, src, dst):                        # CPU single-stepper stands in for the CUDA pass
        assert emu.emu_ntt_slab_gl64(which, src.data_ptr(), dst.data_ptr(), lg, lg_g, rank, 0, 14) == 0

    mine = parallel.ntt_slab(local, lg, 0, pass_fn, all_to_all=False).numpy().view(np.uint64)
    gathered = [torch.empty_like(torch.from_numpy(mine.view(np.int64))) for _ in range(world)]
    dist.all_gather(gathered, torch.from_numpy(mine.view(np.int64).copy()))
    full = parallel.gather_columns([g.numpy().view(np.uint64) for g in gathered], lg, lg_g, s1=s1)
    q.put((rank, bool(np.array_equal(full, o.ntt_gl64(x, o.NN)))))
    dist.destroy_process_group()


@pytest.mark.parametrize("world,lg,split", [(2, 10, None), (4, 12, None), (2, 9, "3,3,3"), (4, 11, "4,3,4")])
def test_slab_sharded_ntt_over_gloo(world, lg, split):
    import subprocess
    import torch.multiprocessing as mp
    so = os.path.join(ROOT, "tests", "emu", "libntt_emu.so")
    if not os.path.exists(so):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", so,
                               os.path.join(ROOT, "tests", "emu", "ntt_emu.cpp")])
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_ntt_worker, args=(r, world, port, lg, q, split)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok in res)
