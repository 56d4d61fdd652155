"""World-size-2 test of the multi-GPU plumbing on CPU (gloo): the unit split
covers every unit exactly once, ranks agree on the max-over-ranks time exactly
as bench.py computes it, and only rank 0 reports.  No kernels run here."""
import os
import socket
import sys

import pytest

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, total_units, out_dir):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    import bench
    from hexl_b200.sharding import rank_block
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    lo, hi = rank_block(total_units, rank, world)
    mine = torch.zeros(total_units, dtype=torch.int64)
    mine[lo:hi] = 1
    dist.all_reduce(mine)                       # every unit owned by exactly one rank
    assert int(mine.min()) == 1 and int(mine.max()) == 1
    t = bench.max_over_ranks(10.0 + rank, world, device="cpu")  # what bench.py does with its event time
    assert t == 10.0 + (world - 1)
    value = bench.whole_job_value(units_per_rank=hi - lo, world=world, seconds=t, weak=False, total_units=total_units)
    assert abs(value - total_units / t) < 1e-9
    if rank == 0:
        open(os.path.join(out_dir, "rank0.txt"), "w").write(f"{value}")
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("total_units", [30, 16, 7])
def test_two_ranks_share_units_and_agree_on_time(tmp_path, total_units):
    import torch.multiprocessing as mp
    port = _free_port()
    mp.spawn(_worker, args=(2, port, total_units, str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "rank0.txt").exists()


def test_split_units_matches_c_abi_rule():
    from hexl_b200.sharding import split_units
    # same arithmetic as csrc/capi.h stage_items: items*d/ndev
    assert split_units(30, 8) == [(0, 3), (3, 7), (7, 11), (11, 15), (15, 18), (18, 22), (22, 26), (26, 30)]
    assert sorted(hi - lo for lo, hi in split_units(30, 8)) == [3, 3, 4, 4, 4, 4, 4, 4]
    for total in (1, 5, 8192):
        for parts in (1, 2, 3, 8):
            blocks = split_units(total, parts)
            assert blocks[0][0] == 0 and blocks[-1][1] == total
            assert all(a[1] == b[0] for a, b in zip(blocks, blocks[1:]))
