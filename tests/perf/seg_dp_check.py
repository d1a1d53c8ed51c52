"""Multi-GPU check of the frame-sharded segmentation trainer (SegTrainer with a process group): the fused
data-parallel optimiser (b200_dp_adam_step over NVLink peer memory) against NCCL all-reduce of
[gradients || losses] + local Adam, and both against a single-GPU trainer holding the whole video, on the same index
batches and initial state.  Parameters must be bit-identical across ranks; the arms must agree to fp32 summation
order (the trip's gradients come from fp32 atomics, so two runs differ in the last bits and Adam can amplify a
near-zero gradient's sign).  Run under torchrun on >= 2 GPUs:

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29534 tests/perf/seg_dp_check.py
"""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))
from b200 import _native as N, atlas as A, seg as SG, synth          # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    H, W, T, B = 96, 160, 16, 4000
    data = synth.throughput_set(H, W, T, seed=0)
    masks = (torch.rand(H, W, T, generator=torch.Generator().manual_seed(2)) < 0.4).float()
    prec = N.PREC_TC if N.lib().b200_device_supports_tc() else N.PREC_FP32
    t0, t1 = A.frame_range(rank, world, T)
    vid = A.DeviceVideo.from_reference_layout(data, dev, t0, t1)
    mask = SG.pack_mask_frames(masks, dev, t0, t1)
    cfg = {"samples_batch": B}
    trainers = {}
    for name, fused in (("nccl", False), ("fused", True)):
        tr = SG.SegTrainer(vid, mask, cfg, precision=prec, device=dev, process_group=dist.group.WORLD, fused_dp=fused)
        torch.manual_seed(0)
        tr.init_like_reference()
        trainers[name] = tr
    assert trainers["fused"]._dp is not None and trainers["nccl"]._dp is None
    whole = SG.SegTrainer(A.DeviceVideo.from_reference_layout(data, dev), SG.pack_mask_frames(masks, dev), cfg,
                          precision=prec, device=dev)
    torch.manual_seed(0)
    whole.init_like_reference()
    out = {"world": world, "precision": "tc" if prec == N.PREC_TC else "fp32"}
    g = torch.Generator().manual_seed(5)
    worst = {"params_fused_nccl": 0.0, "losses_fused_nccl": 0.0, "params_vs_single": 0.0, "losses_vs_single": 0.0}
    counts_ok = True
    for it in (0, 1, 2, 3, 6000, 6001, 10001):
        inds = torch.randint(H * W * T, (B, 1), generator=g)
        res = {name: tr.step_host(inds, it) for name, tr in trainers.items()}
        ref = whole.step_host(inds, it)
        rel = lambda a, b: float(abs(a[:12] - b[:12]).max() / abs(b[0]))
        worst["losses_fused_nccl"] = max(worst["losses_fused_nccl"], rel(res["fused"], res["nccl"]))
        worst["losses_vs_single"] = max(worst["losses_vs_single"], rel(res["nccl"], ref))
        # the count entries hold the global counts on every rank: world * count after the sum
        counts_ok = counts_ok and all(r[12] == world * ref[12] and r[13] == world * ref[13] for r in res.values())
        pf, pn = trainers["fused"].params, trainers["nccl"].params
        worst["params_fused_nccl"] = max(worst["params_fused_nccl"], float((pf - pn).abs().max()))
        worst["params_vs_single"] = max(worst["params_vs_single"], float((pn - whole.params).abs().max()))
    out.update(worst)
    out["counts_ok"] = counts_ok
    # identical parameters on every rank, in both arms
    diffs = []
    for tr in trainers.values():
        ref = tr.params.clone()
        dist.broadcast(ref, 0)
        diffs.append(float((ref - tr.params).abs().max()))
    out["rank_param_diff"] = max(diffs)
    sd = trainers["fused"].optimizer_state_dict()            # collective: assembles the sharded moments
    out["moments_rel"] = float((trainers["fused"].exp_avg - trainers["nccl"].exp_avg).abs().max() /
                               trainers["nccl"].exp_avg.abs().max())
    out["checkpoint_tensors"] = len(sd["state"])
    out["steps"] = [int(trainers[n].step_count) for n in ("nccl", "fused")] + [int(whole.step_count)]
    # 7 Adam steps of lr 1e-4: a parameter moves by <= 7e-4, a flipped near-zero gradient sign by up to twice that
    ok = (out["rank_param_diff"] == 0.0 and counts_ok and worst["losses_fused_nccl"] <= 1e-4 and
          worst["losses_vs_single"] <= 1e-4 and worst["params_fused_nccl"] <= 1.5e-3 and
          worst["params_vs_single"] <= 1.5e-3 and out["moments_rel"] <= 1e-2 and out["steps"] == [7, 7, 7])
    out["ok"] = bool(ok)
    t = torch.tensor([1.0 if ok else 0.0], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        out["all_ranks_ok"] = bool(t.item() == 1.0)
        print(json.dumps(out), flush=True)
    torch.cuda.synchronize(); dist.barrier()
    sys.stdout.flush()
    os._exit(0 if t.item() == 1.0 else 1)


if __name__ == "__main__":
    main()
