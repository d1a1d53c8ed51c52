"""Stage-by-stage check of the wgmma path against the oracle / the fp32 path (run on the GPU box)."""
import os, sys, json, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "all-in-one-deflicker_b200"))
from b200 import _native as N, atlas as A, synth
from oracle import atlas_oracle as O

GOLD = os.path.join(ROOT, "tests", "golden")
DEV = "cuda"

def params():
    z = np.load(os.path.join(GOLD, "params_seed1234.npz"))
    return [torch.from_numpy(z[f"map{i}"]) for i in range(12)], [torch.from_numpy(z[f"atl{i}"]) for i in range(16)]

def ws_views(tr, B, tc):
    cap = (B + 127) // 128 * 128
    ws = tr._workspace()
    base = (ws.data_ptr() + 255) // 256 * 256 - ws.data_ptr()
    r256 = lambda n: (n + 255) // 256 * 256
    off = base + 256
    off_list = off; off += r256(cap * 4)
    off_x = off; off += r256(9 * cap * 16)
    off_t = off; off += r256(cap * 48)
    off_duv = off; off += r256(9 * cap * 8)
    off_dy = off; off += r256(3 * cap * 12)
    off_dpe = off; off += r256(3 * cap * 40 * 4)
    out = dict(cap=cap, x_map=ws[off_x:off_x + 9 * cap * 16].view(torch.float32).view(9 * cap, 4),
               d_uv=ws[off_duv:off_duv + 9 * cap * 8].view(torch.float32).view(9 * cap, 2))
    if tc:
        out["uv"] = ws[off:off + 9 * cap * 8].view(torch.float32).view(9 * cap, 2); off += r256(9 * cap * 8)
        out["y"] = ws[off:off + 3 * cap * 12].view(torch.float32).view(3 * cap, 3)
    return out

def main():
    small = "--big" not in sys.argv and "--mid" not in sys.argv
    mp, ap = params()
    if small:
        z = np.load(os.path.join(GOLD, "iteration.npz"))
        data = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("video_")}
        inds = torch.from_numpy(z["inds"]); B = 64
    elif "--mid" in sys.argv:
        data = synth.throughput_set(60, 100, 9, seed=3)
        B = int(os.environ.get("DIAG_B", "3000"))
        inds = torch.randint(60 * 100 * 9, (B, 1), generator=torch.Generator().manual_seed(2))
    else:
        data = synth.throughput_set(108, 192, 20, seed=0)
        B = 10000
        inds = torch.randint(108 * 192 * 20, (B, 1), generator=torch.Generator().manual_seed(1))
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    res = {}
    grads = {}
    for name, prec in (("fp32", N.PREC_FP32), ("tc", N.PREC_TC)):
        tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=prec, device=DEV)
        tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
        tr.indices.copy_(inds.reshape(-1))
        t0 = time.time()
        tr.loss_grad(True); torch.cuda.synchronize()
        print(name, "loss_grad ok in %.3fs" % (time.time() - t0), "losses", tr.losses.cpu().numpy()[:6])
        grads[name] = tr.grads.clone()
        if prec == N.PREC_TC:
            v = ws_views(tr, B, True)
            x = v["x_map"].cpu()
            with torch.no_grad():
                uv_ref = O.mlp_forward(O.MAPPING_SPEC, mp, x[:, :3])
                y_ref = O.mlp_forward(O.ATLAS_SPEC, ap, uv_ref[:3 * v["cap"]] * 0.5 + 0.5)
            cap = v["cap"]
            live = torch.zeros(9 * cap, dtype=torch.bool)
            for g in range(9): live[g * cap: g * cap + B] = True
            e_uv = (v["uv"].cpu() - uv_ref)[live].abs().max().item()
            e_y = (v["y"].cpu() - y_ref)[live[:3 * cap]].abs().max().item()
            print("TC forward: max|uv err| %.3e  max|y err| %.3e" % (e_uv, e_y))
            res["uv_err"], res["y_err"] = e_uv, e_y
            if e_uv > 1e-3:
                d = (v["uv"].cpu() - uv_ref)
                print("uv sample rows tc:", v["uv"].cpu()[:4], "ref:", uv_ref[:4])
                print("rows with err>1e-3:", int((d.abs().max(1).values > 1e-3).sum()), "of", d.shape[0])
        res[name + "_losses"] = tr.losses.cpu().numpy().tolist()
    # gradient comparison per tensor against a float64 evaluation of the oracle
    video64 = O.Video(**{k: v.double() if v.dtype == torch.float32 else v for k, v in data.items() if k != "clean"})
    mp64 = [p.double().requires_grad_(True) for p in mp]
    ap64 = [p.double().requires_grad_(True) for p in ap]
    terms = O.iteration_losses(video64, mp64, ap64, inds, 0)
    terms["total"].backward()
    truth = [p.grad.float().to(DEV) for p in mp64 + ap64]
    tr = A.AtlasTrainer(vid, {"samples_batch": B}, precision=N.PREC_FP32, device=DEV)
    worst = 0
    i = 0
    for which in ("mapping", "atlas"):
        a = tr._views(grads["fp32"], which); b = tr._views(grads["tc"], which)
        for k in a:
            ref = truth[i]; i += 1
            e32 = (a[k] - ref).abs().max().item(); etc = (b[k] - ref).abs().max().item(); sc = ref.abs().max().item()
            rel = etc / (sc + 1e-30)
            worst = max(worst, rel)
            bad = "  <<<" if etc > max(4 * e32, 2e-5 * sc) else ""
            if b[k].dim() == 2 and bad:
                d = (b[k] - ref).abs()
                rows_bad = (d.max(1).values > 0.1 * etc).sum().item(); cols_bad = (d.max(0).values > 0.1 * etc).sum().item()
                bad += f" rows>{rows_bad} cols>{cols_bad} argmax {divmod(int(d.argmax()), d.shape[1])}"
            print(f"grad {which:8s} {k:18s} max|ref| {sc:.3e} err_fp32 {e32:.3e} err_tc {etc:.3e}{bad}")
    res["worst_grad_rel"] = worst
    print(json.dumps(res))

if __name__ == "__main__":
    main()
