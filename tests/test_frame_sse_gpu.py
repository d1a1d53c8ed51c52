"""b200_frame_sse, the device squared error behind the frame-sharded evaluation's PSNR: float64 sums against numpy at
edge and full frame sizes, on whole-video and frame-shard videos; bit-stable across calls and CUDA-graph replays;
non-resident frames and short workspaces refused; no spills."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "all-in-one-deflicker_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
DEV = "cuda:0"
gpu = pytest.mark.gpu


def _video(H, W, T, t_begin, t_end, seed):
    """A DeviceVideo whose resident records hold random fp32 values in every channel (rgb in 0..2)."""
    g = torch.Generator().manual_seed(seed)
    n = H * W * (t_end - t_begin)
    records = torch.rand(max(n, 1) * N.RECORD_FLOATS, generator=g).to(DEV)
    words = (H * W * T + 31) // 32 + 1
    bits = torch.zeros(words, dtype=torch.int32, device=DEV)
    return A.DeviceVideo(H, W, T, t_begin, t_end, records, bits, bits.clone())


def _numpy_sse(video, f, rgb):
    HW = video.H * video.W
    rec = video.records.cpu().numpy().reshape(-1, N.RECORD_FLOATS)[(f - video.t_begin) * HW:(f - video.t_begin + 1) * HW, :3]
    d = rgb.cpu().numpy().reshape(HW, 3).astype(np.float64) - rec.astype(np.float64)
    return float(np.sum(d * d))


@gpu
@pytest.mark.parametrize("H,W", [(1, 1), (7, 13), (432, 768), (1080, 1920)])
@pytest.mark.parametrize("shard", [False, True])
def test_frame_sse_matches_float64_numpy(H, W, shard):
    T, (t0, t1) = (3, (0, 3)) if not shard else (5, (2, 4))
    video = _video(H, W, T, t0, t1, seed=H * 31 + W)
    g = torch.Generator().manual_seed(W)
    for f in range(t0, t1):
        rgb = torch.rand(H, W, 3, generator=g).to(DEV)
        got = float(A.frame_sse(video, f, rgb).item())
        want = _numpy_sse(video, f, rgb)
        assert abs(got - want) <= 1e-12 * want, (f, got, want)
        # the PSNR of the evaluation, from the same records
        assert abs(A.psnr_device(video, f, rgb) - A.psnr(video.frame_rgb(f).cpu(), rgb.cpu())) < 1e-9


@gpu
def test_frame_sse_is_bit_stable_across_calls_and_graph_replay():
    H, W = 1080, 1920
    video = _video(H, W, 4, 1, 3, seed=9)
    rgb = torch.rand(H, W, 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    first = A.frame_sse(video, 2, rgb).clone()
    for _ in range(5):
        assert torch.equal(A.frame_sse(video, 2, rgb), first)
    out = torch.zeros(1, dtype=torch.float64, device=DEV)
    ws = torch.empty(int(N.lib().b200_frame_sse_workspace_bytes(H, W)), dtype=torch.uint8, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        A.frame_sse(video, 2, rgb, out, ws)               # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        A.frame_sse(video, 2, rgb, out, ws)
    for _ in range(3):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, first)


@gpu
def test_frame_sse_refuses_non_resident_frames_and_short_workspaces():
    lib = N.lib()
    H, W = 7, 13
    video = _video(H, W, 6, 2, 4, seed=1)
    rgb = torch.rand(H, W, 3, device=DEV)
    out = torch.zeros(1, dtype=torch.float64, device=DEV)
    need = int(lib.b200_frame_sse_workspace_bytes(H, W))
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    st = N.current_stream()
    for f in (0, 1, 4, 5, -1):
        assert lib.b200_frame_sse(C.byref(video.struct), f, N.ptr(rgb), N.ptr(out), N.ptr(ws), need, st) == 1
        assert b"not resident" in lib.b200_last_error()
    assert lib.b200_frame_sse(C.byref(video.struct), 2, N.ptr(rgb), N.ptr(out), N.ptr(ws), need - 8, st) == 3
    assert b"workspace too small" in lib.b200_last_error()
    assert lib.b200_frame_sse(C.byref(video.struct), 3, N.ptr(rgb), N.ptr(out), N.ptr(ws), need, st) == 0
    torch.cuda.synchronize()
    with pytest.raises(N.B200Error):
        A.frame_sse(video, 4, rgb)
    assert lib.b200_frame_sse_workspace_bytes(0, 5) == -1


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not available")
def test_frame_sse_kernels_do_not_spill(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(CSRC, "eval_sse.cu"), "-o", str(tmp_path / "eval_sse.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    log = r.stdout + r.stderr
    kernels = re.findall(r"Function properties for (\S*frame_sse\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                         r"stores, (\d+) bytes spill loads", log)
    assert {k for k, *_ in kernels} >= {"_ZN4b20024frame_sse_partial_kernelEPKfS1_lPd",
                                        "_ZN4b20022frame_sse_final_kernelEPKdiPd"}, log
    assert all(int(s) == 0 and int(st) == 0 and int(ld) == 0 for _, s, st, ld in kernels), kernels
