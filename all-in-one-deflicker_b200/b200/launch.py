"""Multi-GPU launch of the flow pre-pass, the stage-1 scripts and stage 2 on one node.

A script started with `--gpus N` (N > 1) and no launcher re-runs itself under `torch.distributed.run`; a script that
finds torchrun's WORLD_SIZE / RANK / LOCAL_RANK joins an NCCL process group on cuda:LOCAL_RANK.  The helpers below are
what every rank of such a run shares: the pair and frame blocks, one random stream, the one-time replica check, the
per-frame values gathered in frame order and the tensors sent point to point to rank 0.  Everything but `init` /
`finish` also runs on a gloo group."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from typing import List, Optional, Tuple

import numpy as np
import torch


def torchrun_env() -> Optional[Tuple[int, int, int]]:
    """(rank, world, local_rank) when the process was started by torch.distributed.run, else None."""
    if "WORLD_SIZE" not in os.environ or "RANK" not in os.environ:
        return None
    return int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))


def relaunch(script: str, argv: List[str], gpus: int) -> int:
    """Run `script argv` on `gpus` ranks of this node under torch.distributed.run and return the launcher's exit code.
    The launcher ends every rank when one fails and then exits non-zero."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(int(gpus)),
           os.path.abspath(script)] + list(argv)
    print(" ".join(cmd), flush=True)
    return subprocess.call(cmd)


def init(local_rank: int):
    """Join the NCCL process group of the launcher on cuda:local_rank.  Returns (device, group)."""
    import torch.distributed as dist
    device = torch.device("cuda", local_rank)
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", device_id=device)
    return device, dist.group.WORLD


def finish():
    """Leave the process group after a run that succeeded on every rank."""
    import torch.distributed as dist
    dist.barrier()
    dist.destroy_process_group()


def pair_block(rank: int, world: int, T: int) -> Tuple[int, int]:
    """Block [p0, p1) of the T - 1 consecutive frame pairs (pair p = frames p, p + 1) whose flows `rank` computes:
    contiguous, split like the frames (frame_range)."""
    from .atlas import frame_range
    return frame_range(rank, world, max(T - 1, 0))


def shared_seed(pg=None) -> int:
    """Seed the global CPU generator of every rank with rank 0's initial seed, so that every rank draws the same
    initialisation, pre-training pixels and index batches.  Collective; returns the seed."""
    import torch.distributed as dist
    obj = [int(torch.initial_seed())]
    dist.broadcast_object_list(obj, src=0, group=pg)
    torch.manual_seed(obj[0])
    return obj[0]


def broadcast_params(params: torch.Tensor, pg=None):
    """Rank 0's parameters on every rank (after each rank's own pre-training).  Collective."""
    import torch.distributed as dist
    dist.broadcast(params, src=0, group=pg)


def digest(t: torch.Tensor) -> str:
    """SHA-256 of a tensor's bytes."""
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def check_replicas(pg=None, **tensors):
    """Raise on every rank if any of `tensors` differs between ranks (compared by checksum).  Collective."""
    import torch.distributed as dist
    mine = {k: digest(v) for k, v in tensors.items()}
    every = [None] * dist.get_world_size(pg)
    dist.all_gather_object(every, mine, group=pg)
    bad = sorted({k for d in every for k in d if d[k] != every[0][k]})
    if bad:
        raise RuntimeError(f"rank {dist.get_rank(pg)}: {', '.join(bad)} differ between ranks; every rank must draw "
                           f"the same random stream")


def gather_frame_values(values, pg=None) -> np.ndarray:
    """Every rank's per-frame values concatenated in rank order, which is frame order (contiguous blocks).
    Collective; every rank receives the merged vector."""
    import torch.distributed as dist
    every = [None] * dist.get_world_size(pg)
    dist.all_gather_object(every, [float(v) for v in values], group=pg)
    return np.asarray([v for vs in every for v in vs], dtype=np.float64)


class Phases:
    """Wall time of a run's phases, each ended on every rank (device synchronised, barrier) before it is read; rank 0
    prints them as one `stage1_phases {...}` JSON line."""

    def __init__(self, pg=None):
        import time
        self.pg, self.clock, self.seconds = pg, time.perf_counter, {}
        self.t = self.clock()

    def mark(self, name: str):
        import torch.distributed as dist
        torch.cuda.synchronize()
        dist.barrier(self.pg)
        now = self.clock()
        self.seconds[name] = self.seconds.get(name, 0.0) + now - self.t
        self.t = now

    def report(self):
        import json
        import torch.distributed as dist
        if dist.get_rank(self.pg) == 0:
            print("stage1_phases " + json.dumps(dict(world=dist.get_world_size(self.pg), **self.seconds)), flush=True)


def collect_on_root(items, counts, numel: int, sink, device, pg=None):
    """Hand every rank's uint8 payloads (`items`: this rank's, flat CPU tensors of `numel` bytes each; `counts`: the
    number each rank holds) to `sink` on rank 0, in rank order and in order within a rank.  Point-to-point over the
    group's backend (device buffers under NCCL).  Collective."""
    import torch.distributed as dist
    rank, world = dist.get_rank(pg), dist.get_world_size(pg)
    on_device = dist.get_backend(pg) == "nccl"
    if rank != 0:
        for t in items:
            dist.send(t.to(device) if on_device else t, dst=0, group=pg)
        if on_device:
            torch.cuda.synchronize(device)
        return
    for t in items:
        sink(t)
    buf = torch.empty(numel, dtype=torch.uint8, device=device if on_device else "cpu")
    for r in range(1, world):
        for _ in range(counts[r]):
            dist.recv(buf, src=r, group=pg)
            sink(buf.to("cpu", copy=True))          # buf is reused for the next payload


def send_to_root(t: torch.Tensor, pg=None):
    """Start sending the device tensor `t` to rank 0: its device buffer under NCCL, a CPU copy under gloo.  Returns
    (work, buffer); the buffer must stay alive and unchanged until work.wait() has returned.  Under NCCL the wait makes
    the current stream wait for the send, so the buffer's memory may then go to later work on that stream."""
    import torch.distributed as dist
    buf = t if dist.get_backend(pg) == "nccl" else t.cpu()
    return dist.isend(buf, dst=0, group=pg), buf


def recv_on_root(shape, src: int, device, pg=None, dtype=torch.float32) -> torch.Tensor:
    """A new `dtype` tensor of `shape` on `device`, received from rank `src` (what it passed to send_to_root): into a
    device buffer under NCCL, whose transfer the current stream then waits for, through a CPU buffer under gloo."""
    import torch.distributed as dist
    on_device = dist.get_backend(pg) == "nccl"
    buf = torch.empty(shape, dtype=dtype, device=device if on_device else "cpu")
    dist.recv(buf, src=src, group=pg)
    return buf if on_device else buf.to(device)
