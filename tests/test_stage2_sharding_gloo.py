"""The sharded stage-2 frame loop (run_frames_sharded of src/neural_filter_and_refinement.py) on gloo process groups,
no GPU: a stub stage whose filter half is a deterministic function of the frame and whose refinement half is a
recurrence over the filter outputs.  For worlds 1-4 and 0, 1, 2, 3 and 7 frames every file is written once, by the
rank that owns it (final files by rank 0), with the contents of the one-process loop; ranks without a frame finish
cleanly."""
import importlib.util
import os
import queue
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from PIL import Image

from b200.stage2 import pad_geometry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FRAME_COUNTS = (0, 1, 2, 3, 7)
H, W = 9, 13                    # padded to 32 x 32: the receiver's shape comes from the header, not from the frame


def _script():
    path = os.path.join(ROOT, "all-in-one-deflicker_b200", "src", "neural_filter_and_refinement.py")
    spec = importlib.util.spec_from_file_location("stage2_script", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class StubStage:
    """Stage2's two halves on the CPU.  filter_png: P_t holds the content frame (plus the atlas frame's mean) inside
    its padding; refine_png: O_t = P_t + 0.5 O_{t-1}.  `filtered` lists the frames this stage filtered."""

    def __init__(self):
        self.filtered = []
        self.reset()

    def reset(self):
        self._o = None

    def filter_png(self, content, atlas):
        h, w = content.shape[:2]
        left, right, _, bottom = pad_geometry(h, w)
        p = torch.zeros(1, 3, h + bottom, w + left + right)
        p[0, :, :h, left:left + w] = torch.from_numpy(content.astype(np.float32)).permute(2, 0, 1) + float(atlas.mean())
        self.filtered.append(int(content[0, 0, 0]))
        return p, {"concat": np.concatenate([content.ravel(), atlas.ravel()]),
                   "filter": p.numpy().view(np.uint8).ravel().copy()}

    def refine_png(self, pred, size):
        left, right, _, bottom = pad_geometry(*size)
        assert tuple(pred.shape) == (1, 3, size[0] + bottom, size[1] + left + right)
        self._o = pred.clone() if self._o is None else pred + 0.5 * self._o
        return self._o.numpy().view(np.uint8).ravel().copy()

    def frame_png(self, content, atlas):
        pred, files = self.filter_png(content, atlas)
        files["final"] = self.refine_png(pred, content.shape[:2])
        return files


def _inputs(folder, T):
    """T content frames (the first pixel is the frame index) and T atlas frames."""
    rng = np.random.default_rng(T)
    cn, an = [], []
    for sub in ("content", "atlas"):
        os.makedirs(os.path.join(folder, sub))
    for t in range(T):
        c = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        c[0, 0, 0] = t
        cn.append(os.path.join(folder, "content", "%05d.png" % t))
        an.append(os.path.join(folder, "atlas", "%05d.png" % t))
        Image.fromarray(c).save(cn[-1])
        Image.fromarray(rng.integers(0, 256, (3, 4, 3), dtype=np.uint8)).save(an[-1])
    return cn, an


def _dirs(root):
    d = {k: os.path.join(root, k) for k in ("concat", "filter", "final")}
    for v in d.values():
        os.makedirs(v, exist_ok=True)
    return d


def _worker(rank, world, port, root, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    script = _script()
    written = []
    write = script._write
    script._write = lambda data, path: (written.append(path), write(data, path))
    out = {}
    try:
        for T in FRAME_COUNTS:
            stage = StubStage()
            base = os.path.join(root, "T%d" % T)
            cn, an = (sorted(os.path.join(base, "in", s, f) for f in os.listdir(os.path.join(base, "in", s)))
                      for s in ("content", "atlas"))
            written.clear()
            script.run_frames_sharded(stage, cn, an, _dirs(os.path.join(base, "w%d" % world)), None, torch.device("cpu"))
            dist.barrier()
            out[T] = {"written": list(written), "filtered": stage.filtered}
    finally:
        dist.destroy_process_group()
    q.put((rank, out))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _read(dirs, T):
    out = {}
    for k, v in dirs.items():
        assert sorted(os.listdir(v)) == ["%05d.png" % t for t in range(T)], k
        out[k] = [open(os.path.join(v, "%05d.png" % t), "rb").read() for t in range(T)]
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_sharded_loop_writes_each_file_once_on_its_owner(world, tmp_path):
    script = _script()
    want = {}
    for T in FRAME_COUNTS:
        base = tmp_path / ("T%d" % T)
        cn, an = _inputs(str(base / "in"), T)
        seq = _dirs(str(base / "seq"))
        script.run_frames(StubStage(), cn, an, seq)
        want[T] = _read(seq, T)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, str(tmp_path), q)) for r in range(world)]
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
    for T in FRAME_COUNTS:
        dirs = {k: str(tmp_path / ("T%d" % T) / ("w%d" % world) / k) for k in ("concat", "filter", "final")}
        assert _read(dirs, T) == want[T], T
        for r in range(world):
            mine = list(range(r, T, world))
            assert res[r][T]["filtered"] == mine, (T, r)
            want_paths = ["%s/%05d.png" % (dirs[k], t) for t in mine for k in ("concat", "filter")]
            if r == 0:
                want_paths += ["%s/%05d.png" % (dirs["final"], t) for t in range(T)]
            assert sorted(res[r][T]["written"]) == sorted(want_paths), (T, r)
