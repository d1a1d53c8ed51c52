"""Stage 2 split across ranks (GPU): Stage2.filter_png / refine_png run as the sharded loop runs them write the files of
the one-GPU loop, byte for byte — emulated in one process for worlds 1-4, in 2 and 3 processes sharing cuda:0 over a
gloo group (the real protocol through the CPU path of b200.launch), the script under torchrun with one rank, and on
two GPUs (the script with --gpus 2, and test.py --gpus 2) where the node has them."""
import glob
import os
import queue
import shutil
import socket
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from b200 import _native as N
from b200 import nn as K
from b200 import stage2 as S2
from test_pipeline_gpu import _write_video
from test_stage2_io_gpu import _dirs, _files, _nets, _script, _sequence

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
DEV = torch.device("cuda:0")


def _precision():
    return "tc" if N.lib().b200_device_supports_tc() else "fp32"


def _emulated(script, st, cn, an, dirs, world):
    """The sharded loop's calls in one process: ranks 1 .. world-1 filter their frames first, rank 0 filters its own
    frames inside the chain and refines copies of every P_t in order."""
    T = len(cn)
    sent = {}
    write = lambda data, key, t: script._write(data, "{}/{:05d}.png".format(dirs[key], t))
    for r in range(1, world):
        for t in range(r, T, world):
            content = script._decode(cn[t])
            pred, files = st.filter_png(content, script._decode(an[t]))
            sent[t] = (pred.clone(), content.shape[:2])
            for k in ("concat", "filter"):
                write(files[k], k, t)
    st.reset()
    for t in range(T):
        if t % world == 0:
            content = script._decode(cn[t])
            pred, files = st.filter_png(content, script._decode(an[t]))
            for k in ("concat", "filter"):
                write(files[k], k, t)
            size = content.shape[:2]
        else:
            pred, size = sent.pop(t)
        write(st.refine_png(pred, size), "final", t)


@pytest.mark.parametrize("precision,dtype", [("tc", np.uint8), ("fp32", np.uint8), ("tc", np.uint16)])
def test_filter_and_refine_in_rank_order_equal_run_frames(precision, dtype, tmp_path):
    if precision == "tc" and not N.lib().b200_device_supports_tc():
        pytest.skip("no tensor-core path on this device")
    K.set_conv_precision(precision)
    try:
        script = _script()
        unet, tn = _nets()
        st = S2.Stage2(unet, tn, DEV)
        for T in (1, 2, 5, 7):
            cn, an = _sequence(str(tmp_path / ("in%d" % T)), T, (75, 133), (23, 37), dtype=dtype)
            ref = _dirs(tmp_path / ("ref%d" % T))
            script.run_frames(st, cn, an, ref)
            want = _files(ref, T)
            for world in (1, 2, 3, 4):
                d = _dirs(tmp_path / ("T%d_w%d" % (T, world)))
                _emulated(script, st, cn, an, d, world)
                assert _files(d, T) == want, (T, world)
        assert want["final"][1] != want["filter"][1]
    finally:
        K.set_conv_precision("tc")


def test_refine_png_refuses_a_p_t_of_another_size():
    K.set_conv_precision(_precision())
    unet, tn = _nets()
    st = S2.Stage2(unet, tn, DEV)
    rng = np.random.default_rng(1)
    pred, _ = st.filter_png(rng.integers(0, 256, (40, 50, 3), dtype=np.uint8),
                            rng.integers(0, 256, (10, 12, 3), dtype=np.uint8))
    assert tuple(pred.shape) == (1, 3, 64, 64)
    for size in ((40, 70), (70, 50)):                 # pads to 64 x 96, 96 x 64
        with pytest.raises(N.B200Error):
            st.refine_png(pred, size)
    with pytest.raises(N.B200Error):
        st.refine_png(pred.cpu(), (40, 50))
    assert st.refine_png(pred, (33, 64)).dtype == np.uint8    # any size that pads to the same shape is accepted


# ---- several processes on cuda:0 over gloo ---------------------------------------------------------------------------
def _worker(rank, world, port, root, precision, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ok = False
    try:
        K.set_conv_precision(precision)
        script = _script()
        unet, tn = _nets()
        cn, an = (sorted(glob.glob(os.path.join(root, "in", s, "*.png"))) for s in ("content", "atlas"))
        dirs = {k: os.path.join(root, "w%d" % world, k) for k in ("concat", "filter", "final")}
        with torch.no_grad():
            script.run_frames_sharded(S2.Stage2(unet, tn, DEV), cn, an, dirs, None, DEV)
        dist.barrier()
        ok = True
    finally:
        dist.destroy_process_group()
        q.put((rank, ok))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_loop_in_processes_sharing_one_gpu_equals_run_frames(world, tmp_path):
    precision = _precision()
    K.set_conv_precision(precision)
    script = _script()
    unet, tn = _nets()
    T = 7
    cn, an = _sequence(str(tmp_path / "in"), T, (75, 133), (23, 37))
    ref = _dirs(tmp_path / "ref")
    with torch.no_grad():
        script.run_frames(S2.Stage2(unet, tn, DEV), cn, an, ref)
    _dirs(tmp_path / ("w%d" % world))
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, str(tmp_path), precision, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {}
    try:
        for _ in range(world):
            r, ok = q.get(timeout=600)
            res[r] = ok
    except queue.Empty:
        pass
    for p in procs:
        p.join(120)
        if p.is_alive():
            p.kill()
            p.join()
    assert all(p.exitcode == 0 for p in procs) and all(res.get(r) for r in range(world)), ([p.exitcode for p in procs], res)
    got = {k: str(tmp_path / ("w%d" % world) / k) for k in ("concat", "filter", "final")}
    assert _files(got, T) == _files(ref, T)


# ---- the script --------------------------------------------------------------------------------------------------
def _checkpoints(work):
    """Random-init stage-2 checkpoints under the reference's names."""
    from src.models.network_filter import UNet
    from src.models.network_local import TransformNet
    os.makedirs(str(work / "pretrained_weights"))
    torch.manual_seed(0)
    torch.save(UNet(in_channels=6, out_channels=3, init_features=32).state_dict(),
               str(work / "pretrained_weights" / "neural_filter.pth"))
    tn = TransformNet(types.SimpleNamespace(nf=32, norm="IN", model="TransformNet", blocks=5), nc_in=12, nc_out=3)
    torch.save(tn.state_dict(), str(work / "pretrained_weights" / "local_refinement_net.pth"))


def _script_inputs(work, vid, T=5, H=72, W=136):
    """Content frames under data/test/<vid>, stand-ins for their stage-1 frames under results/<vid>/stage_1/output
    (blurred copies), and the checkpoints."""
    import cv2
    _write_video(str(work / "data" / "test" / vid), T=T, H=H, W=W)
    out = work / "results" / vid / "stage_1" / "output"
    os.makedirs(str(out))
    for f in sorted(glob.glob(str(work / "data" / "test" / vid / "*.png"))):
        cv2.imwrite(str(out / os.path.basename(f)), cv2.GaussianBlur(cv2.imread(f), (0, 0), 2.0))
    _checkpoints(work)


def _env():
    env = dict(os.environ, PYTHONPATH=PKG, B200_ALLOW_RANDOM_RAFT="1")
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        env.pop(k, None)
    return env


def _run(cmd, cwd, timeout=900):
    r = subprocess.run(cmd, cwd=str(cwd), env=_env(), capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return r


def _stage2_dirs(work, vid):
    res = work / "results" / vid
    return {"concat": str(res / "neural_filter" / "concat"), "filter": str(res / "neural_filter" / "output"),
            "final": str(res / "final" / "output")}


def _same_outputs(a, b, vid, T):
    got, want = _files(_stage2_dirs(a, vid), T), _files(_stage2_dirs(b, vid), T)
    for k in want:
        assert got[k] == want[k], k


SCRIPT = os.path.join(PKG, "src", "neural_filter_and_refinement.py")


def test_script_under_torchrun_with_one_rank_equals_the_plain_script(tmp_path):
    plain, ranked = tmp_path / "plain", tmp_path / "ranked"
    _script_inputs(plain, "clip")
    shutil.copytree(str(plain), str(ranked))
    _run([sys.executable, SCRIPT, "--video_name", "clip"], plain)
    r = _run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", "1", SCRIPT,
              "--video_name", "clip"], ranked)
    assert '"world": 1' in r.stdout and '"frames": 5' in r.stdout, r.stdout[-2000:]
    _same_outputs(ranked, plain, "clip", 5)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="--gpus 2 needs two GPUs on the node")
def test_script_on_two_gpus_equals_the_plain_script(tmp_path):
    plain, two = tmp_path / "plain", tmp_path / "two"
    _script_inputs(plain, "clip", T=7)
    shutil.copytree(str(plain), str(two))
    _run([sys.executable, SCRIPT, "--video_name", "clip"], plain)
    r = _run([sys.executable, SCRIPT, "--video_name", "clip", "--gpus", "2"], two)
    assert '"world": 2' in r.stdout, r.stdout[-2000:]
    _same_outputs(two, plain, "clip", 7)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="test.py --gpus 2 needs two GPUs on the node")
def test_driver_on_two_gpus_writes_the_stage2_files_of_one_gpu(tmp_path):
    """test.py --gpus 2 end to end; then the plain stage-2 script on the same stage-1 output frames."""
    two, plain = tmp_path / "two", tmp_path / "plain"
    _write_video(str(two / "clip"))
    _checkpoints(two)
    shutil.copytree(str(two / "pretrained_weights"), str(plain / "pretrained_weights"))
    _run([sys.executable, os.path.join(PKG, "test.py"), "--video_frame_folder", "clip", "--gpus", "2"], two, 3000)
    shutil.copytree(str(two / "data" / "test" / "clip"), str(plain / "data" / "test" / "clip"))
    shutil.copytree(str(two / "results" / "clip" / "stage_1" / "output"),
                    str(plain / "results" / "clip" / "stage_1" / "output"))
    _run([sys.executable, SCRIPT, "--video_name", "clip"], plain)
    _same_outputs(two, plain, "clip", 6)
