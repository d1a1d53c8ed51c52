"""FusedDp.gather_moments on CPU (gloo, 2 to 4 processes).  Under the fused data-parallel optimiser a rank's Adam
moments are right only on its slice of the parameters (b200_dp_slice) and stale elsewhere.  gather_moments zeroes
everything outside the slice and takes one SUM all-reduce, which must leave the full moments on every rank, bit for
bit.  This is the host half of a checkpoint's Adam state under the fused optimiser; tests/test_optimizer_gpu.py
checks that the kernel writes exactly the owned slices."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG


def _sizes():
    """(n_params, n_total) of the dp table of tests/test_optimizer_gpu.py: both stage-1 buffers with their loss
    vectors, and two tiny buffers whose ranks have empty slices or slices inside the loss tail."""
    atlas = A.AtlasTrainer(None, device="cpu").n_params
    seg = SG.SegTrainer(None, None, device="cpu").n_params
    return [(atlas, atlas + N.LOSS_FLOATS), (seg, seg + N.SEG_LOSS_FLOATS), (4, 4 + N.LOSS_FLOATS),
            (12, 12 + N.LOSS_FLOATS)]


def _owned(world, rank, n_params, n_total):
    """The parameters whose moments `rank` keeps: its slice of the [gradients || losses] buffer, cut at n_params."""
    b, c = C.c_int64(), C.c_int64()
    N.check(N.lib().b200_dp_slice(world, rank, n_total, C.byref(b), C.byref(c)), "b200_dp_slice")
    return min(b.value, n_params), min(b.value + c.value, n_params)


def _full_moments(n_params):
    """The moments every rank must end with, nonzero everywhere so that a missing slice cannot pass as zeros."""
    rng = np.random.default_rng(n_params)
    m = (rng.uniform(0.5, 2.0, n_params) * rng.choice([-1e-3, 1e-3], n_params)).astype(np.float32)
    v = (rng.uniform(0.5, 2.0, n_params) * 1e-6).astype(np.float32)
    return m, v


def _worker(rank, world, port, sizes, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    results = []
    for n_params, n_total in sizes:
        stub = types.SimpleNamespace(world=world, comm=types.SimpleNamespace(rank=rank), n_params=n_params,
                                     n_total=n_total, pg=dist.group.WORLD)
        lo, hi = _owned(world, rank, n_params, n_total)
        rng = np.random.default_rng([rank, n_params])
        full = _full_moments(n_params)
        # what the kernel leaves behind: the right values on the owned slice, stale nonzero values elsewhere
        mine = []
        for ref in full:
            t = (rng.uniform(1.0, 2.0, n_params) * (rank + 1)).astype(np.float32)
            t[lo:hi] = ref[lo:hi]
            mine.append(torch.from_numpy(t))
        A.FusedDp.gather_moments(stub, *mine)
        results.append((n_params, lo, hi, [bool(np.array_equal(t.numpy().view(np.int32), ref.view(np.int32)))
                                           for t, ref in zip(mine, full)]))
    q.put((rank, results))
    dist.destroy_process_group()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("world", [2, 3, 4])
def test_gather_moments_assembles_full_moments(world):
    sizes = _sizes()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000) + 11 * world + 3
    procs = [ctx.Process(target=_worker, args=(r, world, port, sizes, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=240) for _ in range(world))
    for p in procs:
        p.join(60)
    assert all(p.exitcode == 0 for p in procs)
    for n_params, n_total in sizes:
        owned = [_owned(world, r, n_params, n_total) for r in range(world)]
        assert owned[0][0] == 0 and owned[-1][1] == n_params
        assert all(a[1] == b[0] for a, b in zip(owned, owned[1:]))    # the owned slices tile the parameters
    for rank in range(world):
        for n_params, lo, hi, ok in got[rank]:
            assert ok == [True, True], (world, rank, n_params, (lo, hi), "exp_avg / exp_avg_sq")
