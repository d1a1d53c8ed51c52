"""Iterations per second of the stage-1 steps with a position-encoded mapping, on one GPU.

    python tools/pe_mapping_rate.py [--steps 300] [--reps 3] [--fallback-lib OTHER/libb200deflicker.so] [--out DIR]

  single-layer step  AtlasTrainer at the benchmark geometry (768x432, 80 frames, 10000 samples, B200_PREC_TC, replayed
                     graphs, half of the steps with the global rigidity term): the default mapping against a mapping on
                     a 4-frequency positional encoding (use_positional_encoding_mapping1).  Both trainers share the
                     video; the two arms alternate `--reps` times in one process.
  segmentation step  SegTrainer (B200_PREC_TC) with PE 4 on mapping1 and PE 2 on mapping2.  With --fallback-lib, the
                     same step is also timed with that build of the library, e.g. one from before the PE mappings had
                     tensor-core kernels, whose step ran them on the fp32 CUDA-core kernels.  Each library runs in a
                     process of its own (`--reps` windows each).

Prints one JSON line with the card's name and power limit; with --out DIR also writes DIR/pe_mapping_rate.json.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "all-in-one-deflicker_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

H, W, T, BATCH = 432, 768, 80, 10000
PE_ATLAS = {"use_positional_encoding_mapping1": True, "number_of_positional_encoding_mapping1": 4}
PE_SEG = dict(PE_ATLAS, use_positional_encoding_mapping2=True, number_of_positional_encoding_mapping2=2)


def _window(step, n):
    import torch
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        step(i)
    e1.record()
    torch.cuda.synchronize()
    return n / (e0.elapsed_time(e1) / 1000.0)


def atlas_rates(steps, reps, warmup):
    import torch
    from b200 import _native as N, atlas as A, synth
    dev = torch.device("cuda", 0)
    video = A.DeviceVideo.from_reference_layout(synth.throughput_set(H, W, T, seed=0), dev)
    g = torch.Generator().manual_seed(1)
    inds = torch.randint(H * W * T, (16, BATCH), generator=g).to(dev)
    arms = {}
    for name, cfg in (("default mapping", {}), ("PE 4 mapping", PE_ATLAS)):
        tr = A.AtlasTrainer(video, dict(cfg, samples_batch=BATCH), precision=N.PREC_TC, device=dev)
        torch.manual_seed(0)
        tr.init_like_reference()

        def step(i, tr=tr):
            tr.indices.copy_(inds[i % 16])
            tr.step(0 if i < steps // 2 else 6000)
        for i in range(warmup):
            step(0 if i % 2 == 0 else steps - 1)       # captures both graphs
        arms[name] = step
    out = {k: [] for k in arms}
    for _ in range(reps):
        for name, step in arms.items():
            out[name].append(_window(step, steps))
    return out


def seg_rates(steps, reps, warmup, lib_path):
    import torch
    from b200 import _native as N
    if lib_path:
        # another build of the library: bind only the symbols it exports
        N.LIB_PATH = os.path.abspath(lib_path)
        handle = C.CDLL(N.LIB_PATH)
        N.SIGNATURES = {k: v for k, v in N.SIGNATURES.items() if hasattr(handle, k)}
    from b200 import atlas as A, seg as SG, synth
    dev = torch.device("cuda", 0)
    video = A.DeviceVideo.from_reference_layout(synth.throughput_set(H, W, T, seed=0), dev)
    masks = (torch.rand(H, W, T, generator=torch.Generator().manual_seed(2)) < 0.4).float()
    tr = SG.SegTrainer(video, SG.pack_mask_frames(masks, dev), dict(PE_SEG, samples_batch=BATCH), precision=N.PREC_TC,
                       device=dev)
    torch.manual_seed(0)
    tr.init_like_reference()
    codes = [int(N.lib().b200_mlp_tc_architecture(tr.descs[k])) for k in ("mapping1", "mapping2")]
    g = torch.Generator().manual_seed(1)
    inds = torch.randint(H * W * T, (8, BATCH), generator=g).to(dev)

    def step(i):
        tr.indices.copy_(inds[i % 8])
        tr.step(0 if i < steps // 2 else 6000)
    for i in range(warmup):
        step(0 if i % 2 == 0 else steps - 1)
    return {"mapping_tc_codes": codes, "it_per_s": [_window(step, steps) for _ in range(reps)]}


def card():
    import torch
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--fallback-lib", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--seg-only-lib", default=None, help=argparse.SUPPRESS)    # child process: one seg arm
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    if args.seg_only_lib is not None:
        print(json.dumps(seg_rates(args.steps, args.reps, args.warmup, args.seg_only_lib or None)))
        return
    t0 = time.time()
    res = {"card": card(), "geometry": f"{W}x{H}, {T} frames, {BATCH} samples, B200_PREC_TC", "steps_per_window": args.steps}
    res["single_layer_step_it_per_s"] = atlas_rates(args.steps, args.reps, args.warmup)
    torch.cuda.empty_cache()
    seg = {}
    for name, lib in (("this library", ""), ("fallback library", args.fallback_lib)):
        if lib is None:
            continue
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--seg-only-lib", lib, "--steps", str(args.steps // 3),
                            "--reps", str(args.reps), "--warmup", str(args.warmup)], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"seg arm '{name}' failed:\n{r.stderr[-3000:]}")
        seg[name] = json.loads(r.stdout.strip().splitlines()[-1])
    res["seg_step_pe_mappings"] = seg
    res["wall_s"] = round(time.time() - t0, 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pe_mapping_rate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
