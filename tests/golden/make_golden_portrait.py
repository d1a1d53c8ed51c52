"""Pins both stage-1 oracles and the input producer on a PORTRAIT video (H > W) against the reference's own modules,
and freezes ``portrait.npz``, ``seg_portrait.npz`` and ``loader_portrait.npz``.

Run ONLY in the build container (needs /root/reference):

    python tests/golden/make_golden_portrait.py

On a landscape or square video resx == max(resx, resy), so the two normalisations the reference mixes cannot be told
apart: the gradient loss normalises its x+1 / y+1 rows by ``resx`` (loss_utils.py:138-143), everything else (base,
rigidity and flow rows, loss scales, pre-training, render, evaluation maps) by ``larger_dim``.  Here H = 40, W = 26:
the halves are 20 and 13 and differ in every row.  Each stage-1 quantity is also stored as a NEGATIVE CONTROL, the
oracle's result with one normalisation swapped for the other, with its distance from the fixture:
``tests/test_portrait_oracle_golden.py`` proves each control lies far outside the bound the GPU tests apply.
"""
import os
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch
from PIL import Image

OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, OUT)
import make_golden as G  # noqa: E402  (loads the reference's IMLP / loss_utils / unwrap_utils by file path)
import make_golden_seg as GS  # noqa: E402
import make_golden_loader as GL  # noqa: E402
from make_golden_loader_seg import synth_mattes  # noqa: E402
from oracle import atlas_oracle as O  # noqa: E402
from oracle import seg_oracle as S  # noqa: E402
from b200 import synth  # noqa: E402

H, W, T = 40, 26, 6
L = max(H, W)
PICK = 64                      # stored entries per gradient tensor: the first 32 and 32 spread over the rest


def same(a, b, what):
    G.same(a, b, what)


def picks(n):
    """Indices of the stored entries of a flat gradient of n entries (the GPU tests use the same rule)."""
    rest = np.linspace(32, n - 1, PICK - 32).round().astype(np.int64) if n > 32 else np.zeros(0, np.int64)
    return np.concatenate([np.arange(min(n, 32)), rest])


def smooth_video(seed):
    """synth.throughput_set with smooth frames: their forward differences are of the size of the networks' own, so the
    gradient loss depends on the step its x+1 / y+1 rows take (on random frames the image differences swamp it)."""
    data = synth.throughput_set(H, W, T, seed=seed)
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    t = torch.arange(T).float()
    data["frames"] = torch.stack([0.5 + 0.4 * torch.sin(xx[..., None] / 7 + c + 0.3 * t) * torch.cos(yy[..., None] / 9 - c)
                                  for c in range(3)], 2).contiguous()
    data["frames_dx"], data["frames_dy"] = O.image_differences(data["frames"])
    return data


def store_grads(fx, tag, grads):
    for i, g in enumerate(grads):
        gf = g.detach().flatten()
        fx[f"{tag}grad{i}_pick"] = gf[torch.from_numpy(picks(gf.numel()))].numpy()
        fx[f"{tag}grad{i}_sum"] = np.float64(gf.double().sum())
    fx[f"{tag}grad_max"] = np.array([float(g.abs().max()) for g in grads])
    fx[f"{tag}grad_fro"] = np.array([float(g.double().norm()) for g in grads])


def store_control(fx, key, c, cg, got, got_g):
    """A negative control's distance from the fixture: the largest relative change of a loss term, and per gradient
    tensor max|change| and ||change||_F (the tests divide these by their bounds)."""
    fx[key + "_loss"] = max(abs(float(c[k]) - float(got[k])) / abs(float(got[k])) for k in got if float(got[k]) != 0)
    fx[key + "_dmax"] = np.array([float((x - y).abs().max()) for x, y in zip(cg, got_g)])
    fx[key + "_dfro"] = np.array([float((x - y).double().norm()) for x, y in zip(cg, got_g)])


def atlas_losses(video, mp, ap, inds, it, **kw):
    m = [p.clone().requires_grad_(True) for p in mp]
    a = [p.clone().requires_grad_(True) for p in ap]
    terms = O.iteration_losses(video, m, a, inds, it, **kw)
    terms["total"].backward()
    return {k: v.detach() for k, v in terms.items()}, [p.grad for p in m + a]


def reference_atlas(ref_m, ref_a, video, table, inds, it):
    """The loop body of src/stage1_neural_atlas.py:159-227, reference functions only (resx = W, as the script)."""
    for p in list(ref_m.parameters()) + list(ref_a.parameters()):
        p.grad = None
    B = inds.shape[0]
    jif = table[:, inds]
    rgb_cur = video.frames[jif[1, :], jif[0, :], :, jif[2, :]].squeeze(1)
    larger = np.maximum(W, H)
    xyt = torch.cat((jif[0, :] / (larger / 2) - 1, jif[1, :] / (larger / 2) - 1, jif[2, :] / (T / 2.0) - 1), dim=1)
    uv = ref_m(xyt)
    rgb_out = (ref_a(uv * 0.5 + 0.5) + 1.0) * 0.5
    gl = G.ref_loss.get_gradient_loss_single(video.frames_dx, video.frames_dy, jif, ref_m, ref_a, rgb_out, "cpu", W, T)
    rl = (torch.norm(rgb_out - rgb_cur, dim=1) ** 2).mean()
    rig = G.ref_loss.get_rigidity_loss(jif, 1, larger, T, ref_m, uv, "cpu", uv_mapping_scale=0.8)
    terms = dict(gradient=gl, rgb=rl, rigidity=rig)
    total = 1.0 * rig
    if it <= 5000:
        terms["rigidity_global"] = G.ref_loss.get_rigidity_loss(jif, 100, larger, T, ref_m, uv, "cpu",
                                                                uv_mapping_scale=0.8)
        total = total + 5.0 * terms["rigidity_global"]
    fll = G.ref_loss.get_optical_flow_loss(jif, uv, video.flow_bwd, video.mask_bwd, larger, T, ref_m, video.flow_fwd,
                                           video.mask_fwd, 0.8, "cpu", use_alpha=True, alpha=torch.ones(B, 1))
    terms["flow"] = fll
    terms["total"] = total + rl * 5000 + 500.0 * fll + gl * 1000
    terms["total"].backward()
    return {k: v.detach() for k, v in terms.items()}, [p.grad for p in list(ref_m.parameters()) + list(ref_a.parameters())]


def load_params(net, params):
    with torch.no_grad():
        for p, q in zip(net.parameters(), params):
            p.copy_(q)


def atlas_fixture():
    z = np.load(os.path.join(OUT, "params_seed1234.npz"))
    mp = [torch.from_numpy(z[f"map{i}"]) for i in range(12)]
    ap = [torch.from_numpy(z[f"atl{i}"]) for i in range(16)]
    ref_m, ref_a = G.build_reference_nets(0)
    load_params(ref_m, mp)
    load_params(ref_a, ap)
    data = smooth_video(3)
    video = O.Video(**data)
    table = G.ref_unwrap.get_tuples(T, video.frames)
    same(O.pixel_table(T, H, W), table, "pixel table")
    fx = dict(H=H, W=W, T=T, **{"video_" + k: v.numpy() for k, v in data.items()})
    for B in (64, 129):
        inds = torch.randint(table.shape[1], (B, 1), generator=torch.Generator().manual_seed(B))
        fx[f"inds{B}"] = inds.numpy()
        for it in (0, 6000):
            tag = f"B{B}_it{it}_"
            want, want_g = reference_atlas(ref_m, ref_a, video, table, inds, it)
            got, got_g = atlas_losses(video, mp, ap, inds, it)
            assert set(got) == set(want)
            for k in want:
                same(got[k], want[k], f"{tag} loss {k}")
            for i, (a, b) in enumerate(zip(got_g, want_g)):
                same(a, b, f"{tag} grad {i}")
            for k, v in got.items():
                fx[tag + "loss_" + k] = np.float32(v)
            store_grads(fx, tag, got_g)
            # negative controls: the gradient rows normalised by max(W, H) (resx := larger_dim), and every use of
            # larger_dim (base, rigidity and flow rows and the loss scales) replaced by W
            for name, kw in (("resx_larger", dict(resx=L)), ("larger_resx", dict(larger_dim=W))):
                c, cg = atlas_losses(video, mp, ap, inds, it, **kw)
                store_control(fx, f"{tag}ctl_{name}", c, cg, got, got_g)

    # pre-training: two steps of unwrap_utils.py:176-198 (frames 0 and 1 of a 2-frame sweep, rows drawn with
    # randint(resy) then randint(resx)) on the portrait geometry
    Tp = 2
    ref_p, _ = G.build_reference_nets(0)
    load_params(ref_p, mp)
    torch.manual_seed(5)
    G.ref_unwrap.pre_train_mapping(ref_p, Tp, 0.8, resx=W, resy=H, larger_dim=np.maximum(W, H), device="cpu",
                                   pretrain_iters=1)
    torch.manual_seed(5)
    m = [p.clone().requires_grad_(True) for p in mp]
    opt = torch.optim.Adam(m, lr=1e-4)
    losses = []
    for f in range(Tp):
        ys, xs = torch.randint(H, (10000, 1)), torch.randint(W, (10000, 1))
        loss = O.pretrain_losses(m, f, ys, xs, Tp, L, 0.8)
        opt.zero_grad()
        loss.backward()
        if f == 0:
            fx["pre_ys"], fx["pre_xs"] = ys.numpy().astype(np.int16), xs.numpy().astype(np.int16)
            store_grads(fx, "pre_", [p.grad for p in m])
            mc = [p.detach().clone().requires_grad_(True) for p in m]
            ctl = O.pretrain_losses(mc, f, ys, xs, Tp, W, 0.8)
            ctl.backward()
            fx["pre_ctl_W_loss"] = abs(float(ctl.detach()) - float(loss.detach())) / float(loss.detach())
            fx["pre_ctl_W_dmax"] = np.array([float((c.grad - p.grad).abs().max()) for c, p in zip(mc, m)])
        opt.step()
        losses.append(np.float32(loss.detach()))
    for p, q in zip(m, ref_p.parameters()):
        same(p.detach(), q.detach(), "pretrain params")
    fx.update(pre_T=Tp, pre_losses=np.array(losses), pre_w0_head=m[0].detach().flatten()[:64].numpy())

    # render of frame 2 (evaluate.py:640-708) and the u8 image
    f = 2
    with torch.no_grad():
        ys, xs = torch.where(torch.ones(H, W) > 0)
        xyt = torch.cat((xs.unsqueeze(1) / (np.maximum(W, H) / 2) - 1, ys.unsqueeze(1) / (np.maximum(W, H) / 2) - 1,
                         (f / (T / 2.0) - 1) * torch.ones(ys.shape[0], 1)), dim=1)
        ref_img = ((ref_a(ref_m(xyt) * 0.5 + 0.5) + 1) * 0.5).view(H, W, 3)
    img = O.render_frame(mp, ap, f, H, W, T)
    same(img, ref_img, "render")
    u8 = O.to_uint8(img)
    ctl = O.render_frame(mp, ap, f, H, W, T, larger=W)
    fx.update(render_frame=f, render_img=img.numpy(), render_u8=u8,
              render_ctl_W=float((ctl - img).abs().max()),
              render_ctl_W_u8=int((O.to_uint8(ctl) != u8).sum()))

    # evaluation maps (evaluate.py:640-700) of frame 2 and of the last frame
    for f in (2, T - 1):
        ys, xs = torch.where(torch.ones(H, W) > 0)
        with torch.no_grad():
            xyt = torch.cat((xs.unsqueeze(1) / (L / 2) - 1, ys.unsqueeze(1) / (L / 2) - 1,
                             (f / (T / 2.0) - 1) * torch.ones(ys.shape[0], 1)), dim=1)
            uv_r = ref_m(xyt)
            jf = torch.cat((xs.unsqueeze(-1), ys.unsqueeze(-1), torch.ones_like(ys.unsqueeze(-1)) * f), dim=1).T.unsqueeze(-1)
            rig_r = G.ref_loss.get_rigidity_loss(jf, 1, np.maximum(W, H), T, ref_m, uv_r, "cpu", uv_mapping_scale=0.8,
                                                 return_all=True)
            if f < T - 1:
                fl_r = G.ref_loss.get_optical_flow_loss_all(jf, uv_r, np.maximum(W, H), T, ref_m, video.flow_fwd,
                                                            video.mask_fwd, 0.8, "cpu", alpha=torch.ones(ys.shape[0], 1))
            else:
                fl_r = torch.zeros(ys.shape[0])
        uv_o, rig_o, fl_o = O.eval_maps(video, mp, f)
        same(uv_o.reshape(-1, 2), uv_r, "eval uv")
        same(rig_o.reshape(-1), rig_r, "eval rigidity")
        same(fl_o.reshape(-1), fl_r, "eval flow error")
        fx[f"eval_f{f}_uv"], fx[f"eval_f{f}_rig"], fx[f"eval_f{f}_flow"] = uv_o.numpy(), rig_o.numpy(), fl_o.numpy()
        cu, cr, cf = O.eval_maps(video, mp, f, larger=W)
        fx[f"eval_f{f}_ctl_W_uv"] = float((cu - uv_o).abs().max())
        # in units of 2e-3: the evaluation tests bound rigidity by 2e-3 |ref| + 1e-3 and flow error by 2e-3 |ref| + 2e-4
        fx[f"eval_f{f}_ctl_W_rig"] = float(((cr - rig_o).abs() / (rig_o.abs() + 0.5)).max())
        fx[f"eval_f{f}_ctl_W_flow"] = float(((cf - fl_o).abs() / (fl_o.abs() + 0.1)).max())
    fx["eval_frames"] = np.array([2, T - 1])
    np.savez_compressed(os.path.join(OUT, "portrait.npz"), **fx)


def seg_fixture():
    cfg = S.SEG_CONFIG
    ref = GS.build_reference_nets(4321)
    torch.manual_seed(4321)
    nets = S.init_nets()
    for k in GS.ORDER:
        for p, q in zip(nets[k], ref[k].parameters()):
            same(p, q.detach(), f"{k} init")
    B = 64
    data = smooth_video(5)
    video = O.Video(**data)
    masks = GS.seg_masks(H, W, T, 9)
    table = G.ref_unwrap.get_tuples(T, video.frames)
    inds = torch.randint(table.shape[1], (B, 1), generator=torch.Generator().manual_seed(13))
    fx = dict(inds=inds.numpy(), H=H, W=W, T=T, masks=masks.numpy(), init_seed=4321,
              **{"video_" + k: v.numpy() for k, v in data.items()})
    for k in GS.ORDER:
        fx[f"init_{k}_sum"] = np.float64(sum(p.double().sum() for p in nets[k]))

    def mine(it, **kw):
        m = {k: [p.detach().clone().requires_grad_(True) for p in nets[k]] for k in GS.ORDER}
        t = S.seg_iteration_losses(video, masks, m, inds, it, cfg, **kw)
        t["total"].backward()
        return {k: v.detach() for k, v in t.items()}, [p.grad for k in GS.ORDER for p in m[k]]

    for it in (0, 6000, 10001):
        for k in GS.ORDER:
            for p in ref[k].parameters():
                p.grad = None
        rt, _ = GS.reference_iteration(ref, video, masks, table, inds, it, cfg)
        rt["total"].backward()
        got, got_g = mine(it)
        assert set(got) == set(rt)
        for k in rt:
            same(got[k], rt[k].detach(), f"seg it {it} loss {k}")
        for i, (a, q) in enumerate(zip(got_g, [q for k in GS.ORDER for q in ref[k].parameters()])):
            same(a, q.grad, f"seg it {it} grad {i}")
        tag = f"it{it}_"
        for k, v in got.items():
            fx[tag + "loss_" + k] = np.float32(v)
        store_grads(fx, tag, got_g)
        for name, kw in (("resx_larger", dict(resx=L)), ("larger_resx", dict(larger_dim=W))):
            c, cg = mine(it, **kw)
            store_control(fx, f"{tag}ctl_{name}", c, cg, got, got_g)

    # pre-training of mapping1 (the seg script pre-trains both mappings with unwrap_utils.pre_train_mapping)
    Tp = 2
    torch.manual_seed(5)
    G.ref_unwrap.pre_train_mapping(ref["mapping1"], Tp, 0.8, resx=W, resy=H, larger_dim=np.maximum(W, H), device="cpu",
                                   pretrain_iters=1)
    torch.manual_seed(5)
    m = [p.clone().requires_grad_(True) for p in nets["mapping1"]]
    opt = torch.optim.Adam(m, lr=1e-4)
    losses = []
    for f in range(Tp):
        ys, xs = torch.randint(H, (10000, 1)), torch.randint(W, (10000, 1))
        loss = O.pretrain_losses(m, f, ys, xs, Tp, L, 0.8)
        opt.zero_grad(); loss.backward(); opt.step()
        losses.append(np.float32(loss.detach()))
    for p, q in zip(m, ref["mapping1"].parameters()):
        same(p.detach(), q.detach(), "seg pretrain params")
    fx.update(pre_T=Tp, pre_losses=np.array(losses), pre_w0_head=m[0].detach().flatten()[:64].numpy())

    # reconstruction of frame 3 (composite + alpha), with the networks at their initial parameters
    f = 3
    with torch.no_grad():
        ref = GS.build_reference_nets(4321)
        ys, xs = torch.where(torch.ones(H, W) > 0)
        larger = np.maximum(np.int64(W), np.int64(H))
        xyt = torch.cat((xs.unsqueeze(1) / (larger / 2) - 1, ys.unsqueeze(1) / (larger / 2) - 1,
                         (f / (T / 2.0) - 1) * torch.ones(ys.shape[0], 1)), dim=1)
        a = 0.5 * (ref["alpha"](xyt) + 1.0)
        a = a * 0.99
        a = a + 0.001
        c1 = (ref["atlas"](ref["mapping1"](xyt) * 0.5 + 0.5) + 1) * 0.5
        c2 = (ref["atlas"](ref["mapping2"](xyt) * 0.5 - 0.5) + 1) * 0.5
        ref_img = (c1 * a + c2 * (1.0 - a)).view(H, W, 3)
    img, alpha_img = S.render_frame_seg(nets, f, H, W, T)
    same(img, ref_img, "seg render")
    same(alpha_img, a.view(H, W), "seg render alpha")
    ci, ca = S.render_frame_seg(nets, f, H, W, T, larger=W)
    fx.update(render_frame=f, render_img=img.numpy(), render_alpha=alpha_img.numpy(), render_u8=O.to_uint8(img),
              render_ctl_W=float(max((ci - img).abs().max(), (ca - alpha_img).abs().max())),
              render_ctl_W_u8=int((O.to_uint8(ci) != O.to_uint8(img)).sum()))
    np.savez_compressed(os.path.join(OUT, "seg_portrait.npz"), **fx)


def loader_fixture():
    """load_input_data_single / load_input_data at resy x resx = 44 x 30 from 52 x 36 flows: newh/oldh = 0.846 and
    neww/oldw = 0.833, so resize_flow's swapped factors differ from the geometric ones."""
    ref = GL.load_module("ref_unwrap_utils_p", os.path.join(GL.REF, "src/models/stage_1/unwrap_utils.py"))
    mine = GL.load_module("our_unwrap_utils_p",
                          os.path.join(GL.ROOT, "all-in-one-deflicker_b200/src/models/stage_1/unwrap_utils.py"))
    frames, flows = GL.synth_inputs(seed=7, T=4, H=52, W=36)
    mattes = synth_mattes(len(frames), 52, 36, seed=4)
    resy, resx = 44, 30
    with tempfile.TemporaryDirectory() as tmp:
        folder = GL.write_inputs(tmp, "vid", frames, flows)
        seg = Path(tmp) / "vid_seg"
        seg.mkdir()
        for i, m in enumerate(mattes):
            Image.fromarray(m).save(str(seg / ("%05d.png" % i)))
        want = ref.load_input_data_single(resy, resx, 200, folder, True, True, folder.parent, "vid")
        got = mine.load_input_data_single(resy, resx, 200, folder, True, True, folder.parent, "vid")
        want_seg = ref.load_input_data(resy, resx, 200, folder, True, True, folder.parent, "vid")
        got_seg = mine.load_input_data(resy, resx, 200, folder, True, True, folder.parent, "vid")
    for name, a, b in zip(GL.NAMES, want, got):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), name
    for name, a, b in zip(GL.NAMES, want_seg, got_seg):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), name + " (load_input_data)"
    for name, a, b in zip(GL.NAMES, want, want_seg):
        if name != "mask_frames":
            assert torch.equal(a, b), name
    assert want[1].shape == (resy, resx, 3, 4)
    assert 0.05 < float(want[0].mean()) < 0.95, "the consistency masks should hold both values"
    out = {"resy": resy, "resx": resx, "want_seg_mask_frames": want_seg[3].numpy()}
    for i, fr in enumerate(frames):
        out[f"frame{i}"] = fr
    for i, (f12, f21) in enumerate(flows):
        out[f"f12_{i}"], out[f"f21_{i}"] = f12, f21
    for i, m in enumerate(mattes):
        out[f"matte{i}"] = m
    for name, a in zip(GL.NAMES, want):
        out["want_" + name] = a.numpy()
    np.savez_compressed(os.path.join(OUT, "loader_portrait.npz"), **out)


def main():
    torch.set_num_threads(1)      # deterministic summation order inside addmm for the fixtures
    atlas_fixture()
    seg_fixture()
    loader_fixture()
    print("portrait fixtures written to", OUT)


if __name__ == "__main__":
    main()
