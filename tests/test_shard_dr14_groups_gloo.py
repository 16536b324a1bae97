"""CPU, world_size 2 over gloo: album DR rows and peaks across ranks.  Each rank holds a contiguous shard of synthetic DR-14
instances (sparse 8000-bin histograms per channel, window counts, top-two window-peak pairs and true-peak holds), builds the
[G, nch * 8000 + 2] rows and [G, nch, 3] peaks as b200m_dr14_group_reduce lays them out, and shard.allreduce_dr14_groups sums the
rows and gathers the peaks.  The summed rows equal the single-process sum bit for bit, and the top two of the gathered parts equal
the single-process top two, with albums whose tracks sit on both ranks, on one rank only, or on none."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
N_TOTAL, G, NCH = 11, 6, 2
GROUPS = np.array([0, 2, 0, -1, 2, 4, 0, 2, -1, 5, 0])        # albums 0 and 2 span both ranks, 4 and 5 one rank, 1 and 3 none


def _instances():
    """per instance: hist [NCH, 8000] (uint32), windows, pairs [NCH, 2] (h0 >= h1 >= 0), holds [NCH]"""
    rng = np.random.default_rng(21)
    hist = np.zeros((N_TOTAL, NCH, 8000), np.int64)
    for i in range(N_TOTAL):
        for c in range(NCH):
            bins = rng.integers(3000, 8000, 40)
            np.add.at(hist[i, c], bins, rng.integers(1, 9, 40))
    windows = hist[:, 0].sum(1)
    pk = rng.uniform(0.0, 1.2, (N_TOTAL, NCH, 2)).astype(np.float32)
    pk[3] = pk[3, :, ::-1]                                      # a pair equal to another's top: ties across ranks
    pk[7] = pk[2]
    pairs = -np.sort(-pk, axis=2)
    holds = rng.uniform(0.5, 2.0, (N_TOTAL, NCH)).astype(np.float32)
    return hist, windows, pairs, holds


def _top2(vals):
    """the top two of a multiset that holds the fresh pair (0, 0)"""
    v = np.sort(np.concatenate([np.zeros(2, np.float32), np.asarray(vals, np.float32).ravel()]))[::-1]
    return v[0], v[1]


def _local(lo, cnt):
    hist, windows, pairs, holds = _instances()
    rows = np.zeros((G, NCH * 8000 + 2), np.int64)
    peaks = np.zeros((G, NCH, 3), np.float32)
    for a in range(G):
        mem = [i for i in range(lo, lo + cnt) if GROUPS[i] == a]
        for i in mem:
            rows[a, :NCH * 8000] += hist[i].ravel()
            rows[a, -2] += windows[i]
            rows[a, -1] += 1
        for c in range(NCH):
            if mem:
                peaks[a, c, :2] = _top2(pairs[mem, c])
                peaks[a, c, 2] = holds[mem, c].max()
    return rows, peaks


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from meters_lv2_b200 import shard
    lo, cnt = shard.shard_range(N_TOTAL, rank, world)
    rows, peaks = _local(lo, cnt)
    t = torch.from_numpy(rows.astype(np.int32))
    stack = shard.allreduce_dr14_groups(t, torch.from_numpy(peaks))
    assert tuple(stack.shape) == (world, G, NCH, 3)
    if rank == 0:
        q.put((t.numpy().copy(), stack.numpy().copy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_album_dr_equals_single_process():
    sys.path.insert(0, HERE)
    from meters_lv2_b200 import shard
    words = NCH * 8000 + 2
    with pytest.raises(ValueError):
        shard.allreduce_dr14_groups(torch.zeros((G, words), dtype=torch.int64), torch.zeros((G, NCH, 3)))
    with pytest.raises(ValueError):
        shard.allreduce_dr14_groups(torch.zeros((G, words + 1), dtype=torch.int32), torch.zeros((G, NCH, 3)))
    with pytest.raises(ValueError):
        shard.allreduce_dr14_groups(torch.zeros((G, words), dtype=torch.int32), torch.zeros((G + 1, NCH, 3)))
    one = shard.allreduce_dr14_groups(torch.zeros((G, words), dtype=torch.int32), torch.ones((G, NCH, 3)))
    assert tuple(one.shape) == (1, G, NCH, 3)                   # no process group: one part
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    rows, stack = q.get(timeout=240)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    ref_rows, _ = _local(0, N_TOTAL)
    assert ref_rows[[0, 2, 4, 5], -1].min() > 0 and not ref_rows[[1, 3]].any()
    assert np.array_equal(rows, ref_rows.astype(np.int32)), "integer all-reduce of album rows must be bit-exact"
    _, _, pairs, holds = _instances()
    for a in range(G):
        mem = np.nonzero(GROUPS == a)[0]
        for c in range(NCH):
            got = _top2(stack[:, a, c, :2])
            want = _top2(pairs[mem, c]) if mem.size else (0.0, 0.0)
            assert got == want, (a, c, got, want)
            assert stack[:, a, c, 2].max() == (holds[mem, c].max() if mem.size else 0.0), (a, c)
