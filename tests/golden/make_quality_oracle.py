"""Full-schedule quality run of the ORACLE on the CPU (build container, no GPU needed).

    nohup python tests/golden/make_quality_oracle.py > /tmp/quality_oracle.log 2>&1 &

SURVEY.md §8(d) quality set at BASELINE config 2 (80 frames of 768x432: flickering translating
texture, exact flows, consistency masks), the reference's whole stage-1 schedule
(src/stage1_neural_atlas.py:112-255): nn.Linear-style init of both IMLPs from torch.manual_seed(SEED),
`pre_train_mapping` (100 sweeps x 80 frames, unwrap_utils.py:176-198), 10 001 loop trips with 10 000
samples each, then the render of every frame (evaluate.py:640-708) and PSNR against the input video
(evaluate.py:740-743).  The index streams come from torch's global CPU generator in the reference's order,
so the repo's GPU run (tests/perf/quality_vs_oracle.py) consumes the *same* batches.

What is frozen into tests/golden/quality_oracle.npz: per-frame and mean PSNR, the loss terms every 50 trips,
the final parameters of both networks (2.7 MB — every rendered frame can be regenerated from them by the oracle
or by b200_render), and 1/4-scale uint8 thumbnails of three rendered frames.

The run takes a few hours at ~1 it/s; it checkpoints to /tmp every 250 trips and resumes from there.
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))
from oracle import atlas_oracle as O            # noqa: E402
from b200 import synth                          # noqa: E402  (pure numpy/torch data generator)

SEED = 2023
H, W, T = 432, 768, 80
ITERS = int(os.environ.get("QUALITY_ITERS", 10001))
PRE_SWEEPS = int(os.environ.get("QUALITY_PRE_SWEEPS", 100))
THREADS = int(os.environ.get("QUALITY_THREADS", 4))
CKPT = os.environ.get("QUALITY_CKPT", "/tmp/quality_oracle_ckpt.pt")
OUT = os.environ.get("QUALITY_OUT", os.path.join(HERE, "quality_oracle.npz"))


def main():
    torch.set_num_threads(THREADS)
    data = synth.quality_set(H, W, T, seed=0)
    data.pop("clean")
    video = O.Video(**data)
    N = H * W * T

    torch.manual_seed(SEED)
    mp = [p.requires_grad_(True) for p in O.init_mlp(O.MAPPING_SPEC)]
    ap = [p.requires_grad_(True) for p in O.init_mlp(O.ATLAS_SPEC)]
    opt = O.make_optimizer(mp, ap)
    losses = []
    pre_losses = []
    start = 0
    pre_done = False
    if os.path.exists(CKPT):
        ck = torch.load(CKPT, weights_only=False)
        with torch.no_grad():
            for p, q in zip(mp + ap, ck["params"]):
                p.copy_(q)
        pre_done = True
        pre_losses = ck["pre_losses"]
        if ck["opt"] is not None:
            opt.load_state_dict(ck["opt"])
        losses = ck["losses"]
        start = ck["next_iter"]
        torch.set_rng_state(ck["rng"])
        print(f"resumed at loop trip {start}", flush=True)

    def save(next_iter, with_opt=True):
        torch.save(dict(params=[p.detach().clone() for p in mp + ap], opt=opt.state_dict() if with_opt else None,
                        losses=losses, pre_losses=pre_losses, next_iter=next_iter, rng=torch.get_rng_state()),
                   CKPT + ".tmp")
        os.replace(CKPT + ".tmp", CKPT)

    if not pre_done:
        t0 = time.time()
        popt = torch.optim.Adam(mp, lr=1e-4)
        for i in range(PRE_SWEEPS):
            for f in range(T):
                ys = torch.randint(H, (10000, 1))
                xs = torch.randint(W, (10000, 1))
                loss = O.pretrain_losses(mp, f, ys, xs, T, max(W, H), 0.8)
                for p in mp:
                    p.grad = None
                loss.backward()
                popt.step()
            pre_losses.append(float(loss))
            if i % 10 == 0:
                print(f"pretrain sweep {i} loss {float(loss):.6f} ({time.time() - t0:.0f}s)", flush=True)
        save(0, with_opt=False)

    t0 = time.time()
    for i in range(start, ITERS):
        inds = torch.randint(N, (10000, 1))
        terms = O.train_iteration(video, mp, ap, opt, inds, i)
        if i % 50 == 0:
            losses.append((i, terms["total"], terms["rgb"], terms["gradient"], terms["rigidity"],
                           terms.get("rigidity_global", float("nan")), terms["flow"]))
        if i % 250 == 0:
            print(f"trip {i} total {terms['total']:.5f} rgb {terms['rgb']:.6f} "
                  f"({(i - start + 1) / (time.time() - t0):.2f} it/s)", flush=True)
            if i > start:
                save(i + 1)
    save(ITERS)

    ps = np.zeros(T)
    thumbs = {}
    for f in range(T):
        img = O.render_frame([p.detach() for p in mp], [p.detach() for p in ap], f, H, W, T)
        ps[f] = O.psnr(video.frames[:, :, :, f], img)
        if f in (0, T // 2, T - 1):
            thumbs[f] = O.to_uint8(img)[::4, ::4].copy()
        print(f"frame {f} psnr {ps[f]:.3f}", flush=True)
    flat = lambda ps_: np.concatenate([p.detach().numpy().ravel() for p in ps_])
    np.savez_compressed(OUT, seed=SEED, video=np.array([T, H, W]), iters=ITERS, pre_sweeps=PRE_SWEEPS,
                        psnr=ps, psnr_mean=ps.mean(), losses=np.array(losses, dtype=np.float64),
                        pre_losses=np.array(pre_losses), mapping_params=flat(mp), atlas_params=flat(ap),
                        thumb_frames=np.array(sorted(thumbs)), thumbs=np.stack([thumbs[k] for k in sorted(thumbs)]))
    print(f"mean PSNR {ps.mean():.4f} dB -> {OUT}", flush=True)


if __name__ == "__main__":
    main()
