"""Quality gate against the oracle (VERDICT r1 item 1c, BASELINE north_star "output PSNR within 0.1 dB of reference").

The oracle ran the reference's WHOLE stage-1 schedule on the CPU (tests/golden/make_quality_oracle.py: quality set
80 x 432 x 768, pre_train_mapping 100 x 80 steps, 10 001 loop trips, render, PSNR) and its results are frozen in
tests/golden/quality_oracle.npz.  This script runs the same schedule on the GPU through the product path (tensor-core
step, CUDA graphs, tensor-core render) from the same seed — identical initial weights and identical index batches,
drawn from torch's CPU generator in the reference's order — and reports

    psnr_b200 - psnr_oracle            (per frame and mean; the gate is |mean difference| <= 0.1 dB)
    the loss curves side by side        (every 50 trips)
    PSNR between the two reconstructions (the oracle's frames are re-rendered from its final parameters)

    python tests/perf/quality_vs_oracle.py [--iters 10001] [--pre-sweeps 100] > quality_vs_oracle.json
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))
from b200 import _native as N, atlas as A, synth          # noqa: E402
from oracle import atlas_oracle as O                         # noqa: E402  (checker only: fixture layout helpers)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10001)
    ap.add_argument("--pre-sweeps", type=int, default=100)
    ap.add_argument("--fixture", default=os.path.join(ROOT, "tests", "golden", "quality_oracle.npz"))
    ap.add_argument("--precision", default="tc", choices=["tc", "fp32"])
    args = ap.parse_args()
    fx = np.load(args.fixture) if os.path.exists(args.fixture) else None
    seed = int(fx["seed"]) if fx is not None else 2023
    T, H, W = (int(v) for v in fx["video"]) if fx is not None else (80, 432, 768)
    dev = "cuda"
    data = synth.quality_set(H, W, T, seed=0)
    data.pop("clean")
    vid = A.DeviceVideo.from_reference_layout(data, dev)
    prec = N.PREC_TC if args.precision == "tc" else N.PREC_FP32
    tr = A.AtlasTrainer(vid, {}, precision=prec, device=dev)
    torch.manual_seed(seed)
    tr.init_like_reference()
    t0 = time.time()
    tr.pretrain(T, H, W, args.pre_sweeps)
    torch.cuda.synchronize()
    t_pre = time.time() - t0
    losses = []
    npix = H * W * T
    t0 = time.time()
    for i in range(args.iters):
        inds = torch.randint(npix, (10000, 1))
        l = tr.step_host(inds, i)
        if i % 50 == 0:
            losses.append([i] + [float(x) for x in l[:6]])
    torch.cuda.synchronize()
    t_loop = time.time() - t0
    t0 = time.time()
    ps = np.zeros(T)
    recon = []
    for f in range(T):
        img = tr.render_frame(f, H, W, T)
        ps[f] = A.psnr(data["frames"][:, :, :, f], img.cpu())
        recon.append(img)
    torch.cuda.synchronize()
    t_render = time.time() - t0
    out = {"video": [T, H, W], "seed": seed, "iters": args.iters, "pre_sweeps": args.pre_sweeps, "precision": args.precision,
           "psnr_b200_mean": float(ps.mean()), "psnr_b200": [float(x) for x in ps],
           "seconds": {"pretrain": t_pre, "loop": t_loop, "render_and_psnr": t_render},
           "losses_b200": losses}
    if fx is not None and int(fx["iters"]) == args.iters and int(fx["pre_sweeps"]) == args.pre_sweeps:
        po = fx["psnr"]
        out["psnr_oracle_mean"] = float(po.mean())
        out["psnr_diff_mean_db"] = float(ps.mean() - po.mean())
        out["psnr_diff_per_frame_db"] = {"min": float((ps - po).min()), "max": float((ps - po).max())}
        out["gate_0p1_db"] = bool(abs(ps.mean() - po.mean()) <= 0.1)
        lo = fx["losses"]                                  # columns: trip, total, rgb, gradient, rigidity, rigidity_global, flow
        rel = [abs(a[1] - b[1]) / abs(b[1]) for a, b in zip(losses, lo)]
        out["loss_total_rel_diff"] = {"first_20_samples": [float(x) for x in rel[:20]], "max": float(max(rel)),
                                      "median": float(np.median(rel)), "final_b200": losses[-1][1], "final_oracle": float(lo[-1][1])}
        # the oracle's reconstruction, re-rendered from its frozen final parameters on this GPU (fp32 CUDA-core path)
        mp, ap_ = [], []
        off = 0
        for k, n in O.MAPPING_SPEC.layer_dims():
            mp += [torch.from_numpy(fx["mapping_params"][off:off + k * n]).view(n, k)]; off += k * n
            mp += [torch.from_numpy(fx["mapping_params"][off:off + n])]; off += n
        off = 0
        for k, n in O.ATLAS_SPEC.layer_dims():
            ap_ += [torch.from_numpy(fx["atlas_params"][off:off + k * n]).view(n, k)]; off += k * n
            ap_ += [torch.from_numpy(fx["atlas_params"][off:off + n])]; off += n
        tr2 = A.AtlasTrainer(vid, {}, precision=N.PREC_FP32, device=dev)
        tr2.load_state(O.state_dict_of(mp), O.state_dict_of(ap_))
        cross, own = [], []
        for f in range(T):
            img_o = tr2.render_frame(f, H, W, T)
            own.append(A.psnr(data["frames"][:, :, :, f], img_o.cpu()))
            cross.append(A.psnr(img_o.cpu(), recon[f].cpu()))
        out["oracle_rerender_psnr_mean"] = float(np.mean(own))          # must reproduce psnr_oracle_mean
        out["psnr_between_reconstructions_db"] = {"mean": float(np.mean(cross)), "min": float(np.min(cross))}
        th = fx["thumbs"]; tf = fx["thumb_frames"]
        d8 = [int(np.abs((recon[int(f)].cpu().double().numpy() * 255).astype(np.uint8)[::4, ::4].astype(int) - th[k].astype(int)).max())
              for k, f in enumerate(tf)]
        out["thumbnail_max_abs_u8_diff"] = d8
        # the oracle's SECOND run (same seed and index stream, 8 instead of 4 CPU threads = another fp32 summation
        # order): the reference arithmetic's own reproducibility, and this run against the mean of the two
        p2 = os.path.join(os.path.dirname(args.fixture), "quality_oracle_run2_summary.npz")
        if os.path.exists(p2):
            po2 = np.load(p2)["psnr"]
            out["oracle_run2_minus_run1_db"] = float(po2.mean() - po.mean())
            out["psnr_diff_vs_mean_of_oracle_runs_db"] = float(ps.mean() - 0.5 * (po.mean() + po2.mean()))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
