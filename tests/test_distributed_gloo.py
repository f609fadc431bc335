"""CPU, world_size 2 (gloo): the N>1 path of bench.py — contiguous frame shards, no data-path collective,
one gather of fixed-size result records — gives the same records as a single process."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import oracle
from headtrackr_b200 import synth
from headtrackr_b200.parallel import gather_records, shard_range

N_FRAMES, W, H, K = 5, 160, 120, 4


def records_for(frames, blob):
    """(n, 1 + 6K) float64: count, then K rects (x, y, w, h, confidence, neighbors)."""
    out = np.zeros((len(frames), 1 + 6 * K), np.float64)
    for i, f in enumerate(frames):
        res = oracle.detect(f, blob)[:K]
        out[i, 0] = len(res)
        for j, r in enumerate(res):
            out[i, 1 + 6 * j: 7 + 6 * j] = r
    return out


def worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    blob = synth.load_cascade_blob()
    lo, hi = shard_range(N_FRAMES, rank, world)
    frames = [synth.frame(100 + i, W, H, n_faces=1) for i in range(lo, hi)]
    local = torch.from_numpy(records_for(frames, blob))
    counts = [shard_range(N_FRAMES, r, world)[1] - shard_range(N_FRAMES, r, world)[0] for r in range(world)]
    allrec = gather_records(local, counts)
    if rank == 0:
        q.put(allrec.numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_equal_one():
    assert [shard_range(5, r, 2) for r in range(2)] == [(0, 2), (2, 5)]
    assert [shard_range(1024, r, 8) for r in range(8)][-1] == (896, 1024)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    blob = synth.load_cascade_blob()
    want = records_for([synth.frame(100 + i, W, H, n_faces=1) for i in range(N_FRAMES)], blob)
    assert np.array_equal(got, want)
    assert want[:, 0].sum() >= N_FRAMES                           # parity is not vacuous


def loop_worker(rank, world, port, q):
    """bench.py's warm-up loop with SKEWED per-rank clocks: [all_gather, all_reduce] per iteration, exit agreed."""
    import time
    from headtrackr_b200.parallel import agreed
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    dist.barrier()                                   # the group's first collective (connection set-up) stays out of the window
    t_w = time.perf_counter() - 0.05 * rank          # rank 1's clock started 50 ms "earlier": it would leave the loop first
    iters = 0
    rec = torch.full((4,), float(rank))
    while agreed(time.perf_counter() - t_w < 1.0):   # a window long enough for >= 10 iterations on a loaded host
        out = [torch.zeros(4) for _ in range(world)]
        dist.all_gather(out, rec)                    # the step's result gather
        time.sleep(0.005)
        dist.barrier()                               # bench.py's barrier()
        iters += 1
    # what follows the loop in bench.py: a barrier, then steps with gathers - the first collective differs from the loop's
    dist.barrier()
    out = [torch.zeros(4) for _ in range(world)]
    dist.all_gather(out, rec)
    t = torch.tensor([float(iters)])
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    q.put((rank, iters, int(t.item()), [int(o[0]) for o in out]))
    dist.barrier()
    dist.destroy_process_group()


def test_rank_local_loop_exit_is_agreed():
    """A loop that ends on a rank-local clock must end on the same iteration everywhere (bench.py's extra warm-up)."""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=loop_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (r0, i0, m0, g0), (r1, i1, m1, g1) = got
    assert i0 == i1 == m0 == m1 and i0 >= 10           # same iteration count on both ranks, and the loop did run
    assert g0 == g1 == [0, 1]
