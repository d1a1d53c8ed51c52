"""Host side of the multi-GPU stage-1 scripts (b200.launch) on gloo process groups, no GPU: the flow pre-pass's pair
blocks, the random stream every rank shares, the one-time replica check and the per-frame PSNR merged in frame
order."""
import os
import queue

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from b200 import atlas as A
from b200 import launch


@pytest.mark.parametrize("world", range(1, 9))
def test_pair_blocks_cover_every_pair_once(world):
    for T in range(1, 18):
        blocks = [launch.pair_block(r, world, T) for r in range(world)]
        covered = [p for a, b in blocks for p in range(a, b)]
        assert covered == list(range(T - 1)), (world, T, blocks)
        assert max(b - a for a, b in blocks) - min(b - a for a, b in blocks) <= 1


def test_torchrun_env_is_read_from_the_launcher_variables(monkeypatch):
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    assert launch.torchrun_env() is None
    monkeypatch.setenv("WORLD_SIZE", "1")
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("LOCAL_RANK", "0")
    assert launch.torchrun_env() == (0, 1, 0)


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    out = {}
    try:
        # every rank starts from a different generator state; after the broadcast they draw the same stream
        torch.manual_seed(1000 + rank)
        torch.randn(rank + 1)
        seed = launch.shared_seed()
        out["seed"] = seed
        params = torch.empty(257).uniform_(-1, 1)
        inds = torch.randint(10 ** 6, (500, 1))
        launch.check_replicas(parameters=params, first_index_batch=inds)
        out["draw"] = float(params.sum() + inds.sum())
        # a rank that drew a different batch is caught on every rank
        bad = inds.clone()
        if rank == world - 1:
            bad[7, 0] += 1
        try:
            launch.check_replicas(parameters=params, first_index_batch=bad)
            out["mismatch"] = None
        except RuntimeError as e:
            out["mismatch"] = str(e)
        # per-frame PSNR of this rank's frame block, merged in frame order
        T = 11
        t0, t1 = A.frame_range(rank, world, T)
        every = np.random.RandomState(5).uniform(10, 40, T)
        merged = launch.gather_frame_values(every[t0:t1])
        out["merged"] = merged.tolist()
        # payloads reach rank 0 in frame order
        counts = [b - a for a, b in (A.frame_range(r, world, T) for r in range(world))]
        got = []
        items = [torch.full((6,), f, dtype=torch.uint8) for f in range(t0, t1)]
        launch.collect_on_root(items, counts, 6, got.append, "cpu")
        out["collected"] = [int(t[0]) for t in got]
    finally:
        dist.destroy_process_group()
    q.put((rank, out))


@pytest.mark.parametrize("world", [2, 4])
def test_seed_broadcast_replica_check_and_psnr_merge(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000) + 11 * world + 3
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(world):
            r, out = q.get(timeout=240)
            res[r] = out
    except queue.Empty:
        pass
    for p in procs:
        p.join(60)
        if p.is_alive():
            p.kill()
            p.join()
    assert all(p.exitcode == 0 for p in procs) and len(res) == world, [p.exitcode for p in procs]
    assert len({res[r]["seed"] for r in res}) == 1
    assert len({res[r]["draw"] for r in res}) == 1
    for r in res:
        assert res[r]["mismatch"] is not None and "first_index_batch" in res[r]["mismatch"]
        assert "parameters" not in res[r]["mismatch"]
    every = np.random.RandomState(5).uniform(10, 40, 11)
    for r in res:
        assert res[r]["merged"] == every.tolist()
        assert np.mean(res[r]["merged"]) == np.mean(every)
    assert res[0]["collected"] == list(range(11))
    assert all(res[r]["collected"] == [] for r in res if r != 0)
