"""CPU, world_size 2 over gloo: album rows across ranks.  Each rank holds a contiguous shard of the clips (CPU oracle banks stand in
for the GPU banks), sums its members' histograms into the same [G, MIX_WORDS] rows, as b200m_ebu_group_reduce lays them out, and
shard.allreduce_mix sums the rows over the ranks: the result equals the single-process sum bit for bit, with albums whose clips sit
on both ranks, on one rank only, or on none."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
N_TOTAL, G, NB = 9, 5, 120
GROUPS = np.array([0, 2, 0, -1, 2, 4, 0, 2, -1])            # album 0 and 2 span both ranks, 4 one rank, 1 and 3 none


def _rows(e, groups, n_groups, mix_words):
    rows = np.zeros((n_groups, mix_words), np.int64)
    for i, g in enumerate(groups):
        if g >= 0:
            hm, hs, c = e.hist(i)
            rows[g, :751] += hm; rows[g, 752:1503] += hs; rows[g, 1504:1508] += c
    return rows


def _run(lo, cnt):
    import _oracle as O
    import _signals as S
    x = S.white(2 * N_TOTAL, 1024 * NB, seed=77)[2 * lo:2 * (lo + cnt)]
    e = O.Ebu(cnt, 2); e.integr("start")
    for b in range(NB):
        e.process(np.ascontiguousarray(x[:, b * 1024:(b + 1) * 1024]))
    return e


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT); sys.path.insert(0, HERE)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from meters_lv2_b200 import shard
    lo, cnt = shard.shard_range(N_TOTAL, rank, world)
    rows = _rows(_run(lo, cnt), GROUPS[lo:lo + cnt], G, shard.MIX_WORDS)
    t = torch.from_numpy(rows.astype(np.int32))
    assert shard.allreduce_mix(t) is t
    if rank == 0:
        q.put(t.numpy().copy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_album_rows_equal_single_process():
    sys.path.insert(0, HERE)
    from meters_lv2_b200 import shard
    with pytest.raises(ValueError):
        shard.allreduce_mix(torch.zeros((G, shard.MIX_WORDS + 1), dtype=torch.int32))
    with pytest.raises(ValueError):
        shard.allreduce_mix(torch.zeros((G, shard.MIX_WORDS), dtype=torch.int64))
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    rows = q.get(timeout=240)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    ref = _rows(_run(0, N_TOTAL), GROUPS, G, shard.MIX_WORDS)
    assert ref[[0, 2, 4], 1504].min() > 0 and not ref[[1, 3]].any()
    assert np.array_equal(rows, ref.astype(np.int32)), "integer all-reduce of album rows must be bit-exact"
