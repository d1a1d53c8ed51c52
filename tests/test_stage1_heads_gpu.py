"""The kernels between the stage-1 networks, sample by sample against float64: sampling (sample_kernel, both the
whole-video and the frame-sharded instance), the fused loss heads (loss_kernel, pretrain_loss_kernel,
seg_loss_kernel), the segmentation glue (seg_pack_kernel, seg_atlas_in_kernel, seg_chain_kernel), the stand-alone
heads of loss_heads.cu, and the independence of a step from what its workspace held before.

Sampling is restated in fp32 with the kernel's rounding and compared bit for bit.  Slot order is not deterministic
(claimed by atomics on a frame shard, compacted in the flow-match groups), so slots are compared as multisets of
complete per-sample records.

The loss heads are restated in float64 from the device's own network outputs.  Every operation carries a
first-order running-error envelope: it adds |result|, and the envelopes of its inputs propagate through the absolute
partial derivatives.  A device value must lie within  C_ENV * u * envelope  (u = 2^-24, C_ENV = 4) of the float64
value.  The envelope carries the cancellation in the rigidity term's determinant, which a fixed tolerance does not;
separate roundings bound what contraction into FMAs does.  A sample whose branch (det >= 0, n1 > 0, n2 > 0, n > 0)
cannot be decided within its envelope is only required to be finite, and the realistic cases require no such sample.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG
from b200 import synth
from oracle import atlas_oracle as O
from seg_common import load_fixture

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
C_ENV = 4.0
TINY = 2.0 ** -126          # floor of every bound: subnormal results
G_FWD, G_BWD = 5, 6


def f32(x):
    return float(np.float32(x))


# ------------------------------------------------------------------------------------------------ float64 + envelope
class E:
    """float64 value with a first-order running-error envelope (in units of u)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v, self.e = np.broadcast_arrays(np.asarray(v, dtype=np.float64), np.asarray(e, dtype=np.float64))

    @staticmethod
    def w(x):
        return x if isinstance(x, E) else E(x)

    def __add__(self, o):
        o = E.w(o); v = self.v + o.v
        return E(v, self.e + o.e + np.abs(v))

    __radd__ = __add__

    def __sub__(self, o):
        o = E.w(o); v = self.v - o.v
        return E(v, self.e + o.e + np.abs(v))

    def __rsub__(self, o):
        return E.w(o) - self

    def __mul__(self, o):
        o = E.w(o); v = self.v * o.v
        return E(v, np.abs(o.v) * self.e + np.abs(self.v) * o.e + np.abs(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = E.w(o)
        with np.errstate(all="ignore"):
            v = self.v / o.v
            e = self.e / np.abs(o.v) + np.abs(self.v) * o.e / (o.v * o.v) + np.abs(v)
        return E(v, e)

    def __rtruediv__(self, o):
        return E.w(o) / self

    def __neg__(self):
        return E(-self.v, self.e)

    def abs(self):
        return E(np.abs(self.v), self.e)

    def sqrt(self):
        v = np.sqrt(np.maximum(self.v, 0.0))
        with np.errstate(all="ignore"):
            e = np.where(v > 0, self.e / (2 * np.where(v > 0, v, 1.0)), np.sqrt(self.e)) + v
        return E(v, e)

    def log(self):
        with np.errstate(all="ignore"):
            return E(np.log(self.v), self.e / np.abs(self.v) + np.abs(np.log(self.v)))

    def bound(self):
        return C_ENV * U * self.e + TINY

    def undecided(self):
        """|v| within the envelope of 0: the sign (or zero-ness) the device sees is not determined."""
        return (np.abs(self.v) <= C_ENV * U * self.e) & ~((self.v == 0) & (self.e == 0))


def where(c, a, b):
    a, b = E.w(a), E.w(b)
    return E(np.where(c, a.v, b.v), np.where(c, a.e, b.e))


def inv_of(n):
    """fp32 1/n of the kernels, as the exact reciprocal plus its rounding."""
    return E(1.0 / n, 1.0 / n) if n > 0 else E(0.0)


class Ratios:
    """Largest error-to-bound ratio per quantity, and the checks themselves."""

    def __init__(self, name):
        self.name, self.r = name, {}

    def close(self, what, got, ref, ok=None):
        got = np.asarray(got, dtype=np.float64)
        ref_v, bnd = np.broadcast_to(ref.v, got.shape), np.broadcast_to(ref.bound(), got.shape)
        ok = np.ones(got.shape, bool) if ok is None else np.broadcast_to(ok, got.shape)
        assert np.all(np.isfinite(got)), (self.name, what, "non-finite device value")
        err = np.abs(got - ref_v)
        bad = ok & ~(err <= bnd)
        if bad.any():
            i = np.argwhere(bad)[0]
            i = tuple(i)
            raise AssertionError(f"{self.name} {what}: {int(bad.sum())} entries out of bound, first at {i}: device "
                                 f"{got[i]!r} float64 {ref_v[i]!r} bound {bnd[i]!r}")
        if ok.any():
            self.r[what] = max(self.r.get(what, 0.0), float((err[ok] / bnd[ok]).max()))

    def report(self):
        worst = max(self.r.values()) if self.r else 0.0
        print(f"\n[{self.name}] max error/bound {worst:.3f}  " +
              " ".join(f"{k}={v:.3f}" for k, v in sorted(self.r.items())))
        return worst


def vec(a):
    """(x, y) of an [n, 2] array as two exact E."""
    a = np.asarray(a, dtype=np.float64)
    return [E(a[:, 0]), E(a[:, 1])]


# ------------------------------------------------------------------------------------------------ loss_math.h in float64
def rigidity(uv0, uva, uvb, L, s, d, coeff, g0, ga, gb, und):
    """rigidity_term: adds into g0/ga/gb (lists of two E), returns the value; marks undecided branches in und."""
    def sc(x):
        return x * L / 2.0 / s / d
    p, q = sc(uv0[0] - uvb[0]), sc(uv0[0] - uva[0])
    r, t = sc(uv0[1] - uvb[1]), sc(uv0[1] - uva[1])
    S = E(L) / 2.0 / s / d
    A_, Bc, D = p * p + r * r, p * q + r * t, q * q + t * t
    a, dd = A_ + f32(0.001), D + f32(0.001)
    det = a * dd - Bc * Bc
    n1s, n2s = A_ * A_ + 2.0 * Bc * Bc + D * D, a * a + 2.0 * Bc * Bc + dd * dd
    n1, n2 = n1s.sqrt(), n2s.sqrt()
    und |= det.undecided() | n1s.undecided() | n2s.undecided()
    inv_det = 1.0 / det
    value = n1 + n2 * inv_det.abs()
    with np.errstate(all="ignore"):
        in1 = where(n1.v > 0, 1.0 / n1, 0.0)
        in2 = where(n2.v > 0, 1.0 / n2, 0.0)
    sgn = np.where(det.v >= 0, 1.0, -1.0)
    k = n2 * inv_det * inv_det * E(sgn)
    gA = A_ * in1 + (a * in2) * inv_det.abs() - k * dd
    gD = D * in1 + (dd * in2) * inv_det.abs() - k * a
    gB = 2.0 * Bc * in1 + (2.0 * Bc * in2) * inv_det.abs() + k * 2.0 * Bc
    gp, gr = 2.0 * p * gA + q * gB, 2.0 * r * gA + t * gB
    gq, gs = 2.0 * q * gD + p * gB, 2.0 * t * gD + r * gB
    w = coeff * S
    g0[0] = g0[0] + w * (gp + gq); g0[1] = g0[1] + w * (gr + gs)
    gb[0] = gb[0] - w * gp;        gb[1] = gb[1] - w * gr
    ga[0] = ga[0] - w * gq;        ga[1] = ga[1] - w * gs
    return value


def flow(uv0, uvm, L, s, coeff, g0, gm, und, on=None):
    """flow_term on the rows where `on` (all rows if None); the others keep g0 / gm and give 0."""
    ex, ey = uvm[0] - uv0[0], uvm[1] - uv0[1]
    ns = ex * ex + ey * ey
    n = ns.sqrt()
    scale = E(L) / (2.0 * s)
    with np.errstate(all="ignore"):
        inv = where(n.v > 0, 1.0 / n, 0.0)
    w = coeff * scale * inv
    on = np.ones(n.v.shape, bool) if on is None else on
    und |= on & ns.undecided()
    for i, e_ in enumerate((ex, ey)):
        gm[i] = where(on, gm[i] + w * e_, gm[i])
        g0[i] = where(on, g0[i] - w * e_, g0[i])
    return where(on, n * scale, 0.0)


def atlas_head(uv, y, tg, wf, wb, cfg, larger, B, n_f, n_b, ng):
    """sample_loss of loss_math.h.  uv: [9][n][2] rows of each sample (flow groups at their compacted rows), y:
    [3][n][3], tg: [n][12].  Returns (duv [9][2] E, dy [3][3] E, values dict, undecided mask)."""
    n = tg.shape[0]
    und = np.zeros(n, bool)
    L, s = float(larger), f32(cfg.uv_mapping_scale)
    ib = inv_of(B)
    w_rgb, w_grad = E(f32(cfg.rgb_coeff)) * ib, E(f32(cfg.gradient_coeff)) * ib
    dy = [[None] * 3 for _ in range(3)]
    v_rgb, v_grad = E(np.zeros(n)), E(np.zeros(n))
    for ch in range(3):
        o, ox, oy = ((E(y[g][:, ch]) + 1.0) * 0.5 for g in range(3))
        e = o - E(tg[:, ch])
        ex = E(tg[:, 3 + ch]) - (ox - o)
        ey = E(tg[:, 6 + ch]) - (oy - o)
        v_rgb = v_rgb + e * e
        v_grad = v_grad + (ex * ex + ey * ey)
        dy[0][ch] = 0.5 * (w_rgb * 2.0 * e + w_grad * 2.0 * (ex + ey))
        dy[1][ch] = 0.5 * (-w_grad * 2.0 * ex)
        dy[2][ch] = 0.5 * (-w_grad * 2.0 * ey)
    duv = [[E(np.zeros(n)), E(np.zeros(n))] for _ in range(9)]
    U_ = [vec(uv[g]) for g in range(9)]
    rig = rigidity(U_[0], U_[3], U_[4], L, s, f32(cfg.derivative_amount), E(f32(cfg.rigidity_coeff)) * ib,
                   duv[0], duv[3], duv[4], und)
    rigg = E(np.zeros(n))
    if cfg.with_global:
        rigg = rigidity(U_[0], U_[7], U_[8], L, s, f32(cfg.global_derivative_amount),
                        E(f32(cfg.global_rigidity_coeff)) * ib, duv[0], duv[7], duv[8], und)
    ff = flow(U_[0], U_[5], L, s, E(0.5 * f32(cfg.flow_coeff)) * inv_of(n_f), duv[0], duv[5], und, wf)
    fb = flow(U_[0], U_[6], L, s, E(0.5 * f32(cfg.flow_coeff)) * inv_of(n_b), duv[0], duv[6], und, wb)
    return duv, dy, dict(rgb=v_rgb, grad=v_grad, rig=rig, rigg=rigg, ff=ff, fb=fb), und


def block_sum(vals, scale, n_blocks, levels_in_block=8):
    """Sum of per-slot values (E) scaled per block and added with one fp32 atomic per block, in any order."""
    tot_v = float(np.sum(vals.v))
    e = float(np.sum(vals.e)) + (levels_in_block + n_blocks + 2) * float(np.sum(np.abs(vals.v)))
    return E(tot_v, e) * scale


# ------------------------------------------------------------------------------------------------ fixtures / runs
def _golden_video(golden_dir):
    z = np.load(os.path.join(golden_dir, "iteration.npz"))
    return {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("video_")}, torch.from_numpy(z["inds"])


def _params(golden_dir):
    z = np.load(os.path.join(golden_dir, "params_seed1234.npz"))
    return [torch.from_numpy(z[f"map{i}"]) for i in range(12)], [torch.from_numpy(z[f"atl{i}"]) for i in range(16)]


_FULL = {}


def _full_video():
    if "d" not in _FULL:
        _FULL["d"] = synth.throughput_set(432, 768, 80, seed=0)
    return _FULL["d"]


def _with_masks(data, mode):
    if mode == "mixed":
        return data
    d = dict(data)
    fill = 0.0 if mode == "zero" else 1.0
    d["mask_fwd"] = torch.full_like(data["mask_fwd"], fill)
    d["mask_bwd"] = torch.full_like(data["mask_bwd"], fill)
    return d


def _atlas_trainer(data, golden_dir, B, prec, pe, t0=0, t1=None):
    vid = A.DeviceVideo.from_reference_layout(data, DEV, t0, t1)
    conf = {"samples_batch": B}
    if pe:
        conf.update(use_positional_encoding_mapping1=True, number_of_positional_encoding_mapping1=pe)
    tr = A.AtlasTrainer(vid, conf, precision=prec, device=DEV)
    if pe:
        torch.manual_seed(11)
        tr.init_like_reference()
    else:
        mp, ap = _params(golden_dir)
        tr.load_state(O.state_dict_of(mp), O.state_dict_of(ap))
    return tr


def _atlas_cfg(tr, B, with_global, colour=True):
    cfg = tr._config(with_global)
    cfg.batch = B
    if not colour:
        cfg.rgb_coeff = 0.0
        cfg.gradient_coeff = 0.0
    return cfg


def _atlas_step(tr, cfg, inds, fill):
    """One b200_atlas_loss_grad_for on a fresh workspace whose bytes are all `fill`; returns the workspace."""
    nbytes = int(tr.lib.b200_atlas_workspace_bytes_for(C.byref(cfg), C.byref(tr.map_desc)))
    ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=DEV)
    idx = inds.reshape(-1).to(DEV)
    N.check(tr.lib.b200_atlas_loss_grad_for(C.byref(cfg), C.byref(tr.map_desc), C.byref(tr.video.struct), N.ptr(idx),
                                            N.ptr(tr.params), N.ptr(tr.grads), N.ptr(tr.losses), N.ptr(ws), ws.numel(),
                                            N.current_stream()), "b200_atlas_loss_grad_for")
    torch.cuda.synchronize()
    return ws


def _atlas_views(tr, cfg, ws):
    off = (C.c_int64 * 8)()
    N.check(tr.lib.b200_atlas_workspace_offsets_for(C.byref(cfg), C.byref(tr.map_desc), N.ptr(ws), off))
    cap = (cfg.batch + 127) // 128 * 128

    def f(o, *shape):
        n = int(np.prod(shape))
        return ws[o:o + 4 * n].view(torch.float32).cpu().numpy().reshape(shape)
    return dict(cap=cap, counters=ws[off[0]:off[0] + 32].view(torch.int32).cpu().numpy(),
                x_map=f(off[2], 9, cap, 4), targets=f(off[3], cap, 12), d_uv=f(off[4], 9, cap, 2),
                d_y=f(off[5], 3, cap, 3), uv=f(off[6], 9, cap, 2), y=f(off[7], 3, cap, 3))


# ------------------------------------------------------------------------------------------------ sampling restated
def _records(data, inds):
    """Per sample of the global batch: t, y, x and the 15 record floats (reference layouts)."""
    H, W, _, T = data["frames"].shape
    n = inds.reshape(-1).numpy()
    t, y, x = n // (H * W), (n // W) % H, n % W
    rec = np.zeros((n.size, 15), np.float32)
    rec[:, 0:3] = data["frames"].numpy()[y, x, :, t]
    rec[:, 3:6] = data["frames_dx"].numpy()[y, x, :, t]
    rec[:, 6:9] = data["frames_dy"].numpy()[y, x, :, t]
    rec[:, 9:11] = data["flow_fwd"].numpy()[y, x, :, t, 0]
    rec[:, 11:13] = data["flow_bwd"].numpy()[y, x, :, t, 0]
    rec[:, 13] = data["mask_fwd"].numpy()[y, x, t, 0]
    rec[:, 14] = data["mask_bwd"].numpy()[y, x, t, 0]
    return t, y, x, rec


def _norm(v, h):
    return (np.float32(v) / np.float32(h)) - np.float32(1.0)


def _rows(t, y, x, rec, H, W, T, resx, d_local, d_global):
    """The nine coordinate rows of sample_kernel in fp32 (xyz only)."""
    larger = max(W, H)
    hL, hX, hT = np.float32(larger / 2.0), np.float32(resx / 2.0), np.float32(T / 2.0)
    fx, fy, ft = x.astype(np.float32), y.astype(np.float32), t.astype(np.float32)
    dl, dg = np.float32(d_local), np.float32(d_global)
    tn = _norm(ft, hT)
    one = np.float32(1.0)
    rows = [
        (_norm(fx, hL), _norm(fy, hL), tn),
        (_norm(fx + one, hX), _norm(fy, hX), tn),
        (_norm(fx, hX), _norm(fy + one, hX), tn),
        (_norm(fx, hL), _norm(fy - dl, hL), tn),
        (_norm(fx - dl, hL), _norm(fy, hL), tn),
        (_norm(fx + rec[:, 9], hL), _norm(fy + rec[:, 10], hL), _norm(ft + one, hT)),
        (_norm(fx + rec[:, 11], hL), _norm(fy + rec[:, 12], hL), _norm(ft - one, hT)),
        (_norm(fx, hL), _norm(fy - dg, hL), tn),
        (_norm(fx - dg, hL), _norm(fy, hL), tn),
    ]
    return np.stack([np.stack(r, axis=1).astype(np.float32) for r in rows])        # [9][n][3]


def _sorted_bits(recs):
    b = np.ascontiguousarray(recs.astype(np.float32)).view(np.uint32)
    return b[np.lexsort(b.T[::-1])] if b.shape[0] else b


def check_sampling(v, data, inds, cfg, ng, t0, t1, matte=None):
    """(a): counts, the multiset of per-sample records, the compaction bijection and the zero padding.  Returns
    (local sample positions in batch order, pf, pb of each local slot) for the loss-head check."""
    H, W, _, T = data["frames"].shape
    B, cap = cfg.batch, v["cap"]
    t, y, x, rec = _records(data, inds)
    rows = _rows(t, y, x, rec, H, W, T, cfg.resx, cfg.derivative_amount, cfg.global_derivative_amount)
    local = (t >= t0) & (t < t1)
    wf, wb = rec[:, 13] != 0, rec[:, 14] != 0
    cnt = v["counters"]
    n_local, n_lf, n_lb = int(local.sum()), int((local & wf).sum()), int((local & wb).sum())
    assert [int(cnt[0]), int(cnt[1]), int(cnt[2]), int(cnt[5]), int(cnt[6])] == \
        [n_local, int(wf.sum()), int(wb.sum()), n_lf, n_lb]
    keep = [g for g in range(ng) if g not in (G_FWD, G_BWD)]
    # reference records: non-flow rows, targets 0-8, matte, flags, flow rows (zero when the flow is invalid)
    li = np.nonzero(local)[0]
    mt = np.zeros(B, np.float32) if matte is None else matte
    ref = np.concatenate([rows[keep][:, li].transpose(1, 0, 2).reshape(li.size, 3 * len(keep)), rec[li, 0:9], mt[li, None],
                          wf[li, None].astype(np.float32), wb[li, None].astype(np.float32),
                          np.where(wf[li, None], rows[G_FWD, li], 0), np.where(wb[li, None], rows[G_BWD, li], 0)],
                         axis=1)
    xm, tg = v["x_map"], v["targets"]
    pf, pb = tg[:n_local, 9].astype(np.int64) - 1, tg[:n_local, 10].astype(np.int64) - 1
    assert np.array_equal(tg[:n_local, 9], np.round(tg[:n_local, 9])) and pf.min(initial=-1) >= -1
    # columns 9 / 10 map the valid samples bijectively onto [0, n_lf) / [0, n_lb)
    assert sorted(pf[pf >= 0].tolist()) == list(range(n_lf)) and sorted(pb[pb >= 0].tolist()) == list(range(n_lb))
    got = np.concatenate([xm[keep][:, :n_local, :3].transpose(1, 0, 2).reshape(n_local, 3 * len(keep)), tg[:n_local, 0:9],
                          tg[:n_local, 11:12], (pf >= 0)[:, None].astype(np.float32), (pb >= 0)[:, None].astype(np.float32),
                          np.where((pf >= 0)[:, None], xm[G_FWD, np.maximum(pf, 0), :3], 0),
                          np.where((pb >= 0)[:, None], xm[G_BWD, np.maximum(pb, 0), :3], 0)], axis=1)
    assert np.array_equal(_sorted_bits(got), _sorted_bits(ref)), "slot records differ from the fp32 restatement"
    # padding: every row the networks may read past the sampled ones is zero, and the fourth column everywhere
    assert np.all(xm[:ng, :, 3] == 0)
    for g in range(ng):
        lim = n_lf if g == G_FWD else (n_lb if g == G_BWD else n_local)
        assert np.all(xm[g, lim:] == 0), f"x_map group {g} rows [{lim}, {cap}) are not zero"
    if t0 == 0 and t1 == T:
        assert np.all(tg[B:] == 0)
    return pf, pb


def check_atlas_head(v, cfg, larger, ng, pf, pb, losses, prec, colour, rt):
    """(b): d_y, d_uv of groups 3..ng-1 (and 0-2 without colour terms), padding rows, the loss vector and the two
    gradient-scale words, from the device's own network outputs."""
    cap, cnt = v["cap"], v["counters"]
    n_local, n_f, n_b = int(cnt[0]), int(cnt[1]), int(cnt[2])
    B = cfg.batch
    s = np.arange(n_local)
    rows = [np.maximum(pf, 0) if g == G_FWD else (np.maximum(pb, 0) if g == G_BWD else s) for g in range(9)]
    uv = np.stack([np.where((g < ng) & ((g != G_FWD) | (pf >= 0)) & ((g != G_BWD) | (pb >= 0)),
                            v["uv"][g, rows[g]].T, 0).T for g in range(9)])
    y = v["y"][:, :n_local]
    duv, dy, vals, und = atlas_head(uv, y, v["targets"][:n_local], pf >= 0, pb >= 0, cfg, larger, B, n_f, n_b, ng)
    ok = ~und
    rt.r["undecided"] = float(und.sum())
    for g in range(3):
        for c in range(3):
            rt.close(f"d_y{g}", v["d_y"][g, :n_local, c], dy[g][c], ok)
    groups = range(3, ng) if colour else range(ng)
    for g in groups:
        for c in range(2):
            if g in (G_FWD, G_BWD):
                p = pf if g == G_FWD else pb
                sel = p >= 0
                rt.close(f"d_uv{g}", v["d_uv"][g, p[sel], c], E(duv[g][c].v[sel], duv[g][c].e[sel]), ok[sel])
            else:
                rt.close(f"d_uv{g}", v["d_uv"][g, :n_local, c], duv[g][c], ok)
    # padding rows of the loss head's own outputs
    assert np.all(v["d_y"][:, n_local:] == 0)
    for g in range(3, ng):
        lim = int(cnt[5]) if g == G_FWD else (int(cnt[6]) if g == G_BWD else n_local)
        assert np.all(v["d_uv"][g, lim:] == 0), f"d_uv group {g} rows [{lim}, {cap}) are not zero"
    # loss vector
    nb = (cap + 127) // 128
    ib = inv_of(B)
    l_rgb, l_grad = block_sum(vals["rgb"], ib, nb), block_sum(vals["grad"], ib, nb)
    l_rig, l_rigg = block_sum(vals["rig"], ib, nb), block_sum(vals["rigg"], ib, nb)
    l_flow = 0.5 * (block_sum(vals["ff"], inv_of(n_f), nb) + block_sum(vals["fb"], inv_of(n_b), nb))
    tot = (E(f32(cfg.rigidity_coeff)) * l_rig + E(f32(cfg.global_rigidity_coeff) if cfg.with_global else 0.0) * l_rigg
           + E(f32(cfg.rgb_coeff)) * l_rgb + E(f32(cfg.flow_coeff)) * l_flow + E(f32(cfg.gradient_coeff)) * l_grad)
    tot = E(tot.v, tot.e + nb * abs(tot.v))
    assert losses[6] == n_f and losses[7] == n_b
    if und.any():
        assert np.all(np.isfinite(losses[1:5]))
    else:
        for i, (name, ref) in enumerate((("loss_rgb", l_rgb), ("loss_grad", l_grad), ("loss_rig", l_rig),
                                         ("loss_rigg", l_rigg)), start=1):
            rt.close(name, losses[i], ref)
    if n_f == 0 or n_b == 0:
        assert np.isnan(losses[5]) and np.isnan(losses[0])
    elif not und.any():
        rt.close("loss_flow", losses[5], l_flow)
        rt.close("loss_total", losses[0], tot)
    # gradient-scale words: a max does not depend on order
    assert int(cnt[3]) == int(np.float32(np.abs(v["d_y"]).max()).view(np.int32)), "counters[3] != bits of max|d_y|"
    after = np.float32(np.abs(v["d_uv"][:ng]).max())
    c4 = float(np.asarray(cnt[4:5], np.int32).view(np.float32)[0])
    if not colour:
        assert int(cnt[4]) == int(after.view(np.int32)), "counters[4] != bits of max|d_uv| (loss head only)"
        return
    head_v = np.max([np.abs(duv[g][c].v[ok]).max(initial=0.0) for g in range(ng) for c in range(2)])
    head_b = np.max([duv[g][c].bound()[ok].max(initial=0.0) for g in range(ng) for c in range(2)])
    assert c4 >= float(np.abs(v["d_uv"][3:ng]).max())
    if prec == N.PREC_TC:
        assert c4 >= float(after)
        if c4 == float(after):
            return
    if not und.any():
        assert abs(c4 - head_v) <= head_b, (c4, head_v, head_b)


# ------------------------------------------------------------------------------------------------ (a) + (b): atlas step
CASES = [
    # name, video, B, precision, with_global, pe, masks, world
    ("fixture-fp32-global", "golden", 64, N.PREC_FP32, True, 0, "mixed", 1),
    ("fixture-tc-global", "golden", 64, N.PREC_TC, True, 0, "mixed", 1),
    ("fixture-fp32-local-2shard", "golden", 64, N.PREC_FP32, False, 0, "mixed", 2),
    ("fixture-tc-local-3shard", "golden", 64, N.PREC_TC, False, 0, "mixed", 3),
    ("B1-fp32-3shard", "golden", 1, N.PREC_FP32, True, 0, "mixed", 3),
    ("B1-tc", "golden", 1, N.PREC_TC, True, 0, "one", 1),
    ("B31-tc-noflow", "golden", 31, N.PREC_TC, True, 0, "zero", 1),
    ("B127-fp32-allflow", "golden", 127, N.PREC_FP32, False, 0, "one", 1),
    ("B128-tc-allflow-2shard", "golden", 128, N.PREC_TC, True, 0, "one", 2),
    ("B129-fp32-pe4-3shard", "golden", 129, N.PREC_FP32, True, 4, "mixed", 3),
    ("B129-tc-pe4", "golden", 129, N.PREC_TC, True, 4, "mixed", 1),
    ("B129-fp32-noflow-2shard", "golden", 129, N.PREC_FP32, False, 0, "zero", 2),
    ("full-B10000-tc", "full", 10000, N.PREC_TC, True, 0, "mixed", 1),
    ("full-B16384-fp32-2shard", "full", 16384, N.PREC_FP32, True, 0, "mixed", 2),
    ("full-B16384-tc-pe4-3shard", "full", 16384, N.PREC_TC, False, 4, "mixed", 3),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_atlas_sampling_and_loss_head(golden_dir, case):
    name, kind, B, prec, wg, pe, masks, world = case
    if prec == N.PREC_TC and not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")
    if kind == "golden":
        data, finds = _golden_video(golden_dir)
        inds = finds[:B] if B <= finds.shape[0] else \
            torch.randint(int(np.prod(data["frames"].shape)) // 3, (B, 1), generator=torch.Generator().manual_seed(B))
    else:
        data = _full_video()
        inds = torch.randint(432 * 768 * 80, (B, 1), generator=torch.Generator().manual_seed(B))
    data = _with_masks(data, masks)
    H, W, _, T = data["frames"].shape
    ng = 9 if wg else 7
    worst = 0.0
    for r in range(world):
        t0, t1 = A.frame_range(r, world, T) if world > 1 else (0, T)
        tr = _atlas_trainer(data, golden_dir, B, prec, pe, t0, t1)
        for colour in (True, False):
            cfg = _atlas_cfg(tr, B, wg, colour)
            ws = _atlas_step(tr, cfg, inds, 0xFF)
            v = _atlas_views(tr, cfg, ws)
            rt = Ratios(f"{name} shard {r}/{world} {'full' if colour else 'no-colour'}")
            pf, pb = check_sampling(v, data, inds, cfg, ng, t0, t1)
            check_atlas_head(v, cfg, max(H, W), ng, pf, pb, tr.losses.cpu().numpy(), prec, colour, rt)
            assert np.all(np.isfinite(tr.grads.cpu().numpy()))
            if kind == "full" or masks == "mixed":
                assert rt.r["undecided"] == 0, "realistic case with undecidable branches"
            rt.r.pop("undecided")
            worst = max(worst, rt.report())
            del ws
        del tr
    torch.cuda.empty_cache()
    assert worst <= 1.0


@pytest.mark.parametrize("prec", [N.PREC_FP32, N.PREC_TC], ids=["fp32", "tc"])
def test_mapping_scale_word_covers_the_flow_groups(golden_dir, prec):
    """counters[4] must see the flow-match groups.  flow_term gives every flow row a gradient of magnitude w (w times
    a unit vector) and the base row its mirror plus the other terms, so in ordinary batches the base group holds the
    maximum of |d_uv| and a scale word that skipped groups 5 / 6 would still be right.  Here only one sample has a valid
    forward flow (n_f = 1: its row weighs n_b times a backward row), chosen so that each component of its backward
    residual opposes its forward one: the two flow terms of its base row cancel in part, and the forward row holds the
    strict maximum.  No colour and no rigidity terms, so d_uv after the step is the loss head's alone in both
    precisions."""
    if prec == N.PREC_TC and not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")
    data, inds = _golden_video(golden_dir)
    B = inds.shape[0]
    H, W, _, T = data["frames"].shape
    both = _with_masks(data, "one")
    tr = _atlas_trainer(both, golden_dir, B, prec, 0)
    cfg = _atlas_cfg(tr, B, False, colour=False)
    cfg.rigidity_coeff = 0.0
    cfg.global_rigidity_coeff = 0.0
    # first step, every flow valid: the forward and backward residuals of every sample
    v = _atlas_views(tr, cfg, _atlas_step(tr, cfg, inds, 0))
    pf, pb = v["targets"][:B, 9].astype(np.int64) - 1, v["targets"][:B, 10].astype(np.int64) - 1
    u0 = v["uv"][0, :B].astype(np.float64)
    uf, ub = v["uv"][G_FWD, pf] - u0, v["uv"][G_BWD, pb] - u0
    n = inds.reshape(-1).numpy()
    unique = np.array([np.count_nonzero(n == k) == 1 for k in n])
    opposed = np.all(uf * ub < 0, axis=1) & unique
    assert opposed.any(), "no sample with opposed residuals in the batch"
    cos = np.sum(uf * ub, axis=1) / (np.linalg.norm(uf, axis=1) * np.linalg.norm(ub, axis=1))
    s0 = int(np.argmin(np.where(opposed, cos, np.inf)))
    # second step: the forward flow valid at s0's pixel only (the records and the bitmaps both come from mask_fwd)
    t, y, x = n[s0] // (H * W), (n[s0] // W) % H, n[s0] % W
    one_fwd = dict(both)
    one_fwd["mask_fwd"] = torch.zeros_like(both["mask_fwd"])
    one_fwd["mask_fwd"][y, x, t, 0] = 1.0
    tr = _atlas_trainer(one_fwd, golden_dir, B, prec, 0)
    v = _atlas_views(tr, cfg, _atlas_step(tr, cfg, inds, 0xFF))
    cnt = v["counters"]
    assert [int(cnt[1]), int(cnt[2]), int(cnt[5]), int(cnt[6])] == [1, B, 1, B]
    rt = Ratios(f"flow-row maximum {'tc' if prec else 'fp32'}")
    pf, pb = check_sampling(v, one_fwd, inds, cfg, 7, 0, T)
    check_atlas_head(v, cfg, max(H, W), 7, pf, pb, tr.losses.cpu().numpy(), prec, False, rt)
    mx = [float(np.abs(v["d_uv"][g]).max()) for g in range(7)]
    assert mx[G_FWD] > max(m for g, m in enumerate(mx) if g != G_FWD), mx
    assert int(cnt[4]) == int(np.float32(mx[G_FWD]).view(np.int32))
    rt.r.pop("undecided")
    assert rt.report() <= 1.0


# ------------------------------------------------------------------------------------------------ (c) pretraining
@pytest.mark.parametrize("prec", [N.PREC_FP32, N.PREC_TC], ids=["fp32", "tc"])
@pytest.mark.parametrize("B", [1, 129, 10000])
def test_pretrain_rows_and_head(golden_dir, prec, B):
    if prec == N.PREC_TC and not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")
    data, _ = _golden_video(golden_dir)
    tr = _atlas_trainer(data, golden_dir, 64, prec, 0)
    H, W, T, f = 432, 768, 80, 37
    larger = max(H, W)
    g = torch.Generator().manual_seed(B)
    ys, xs = torch.randint(H, (B,), generator=g), torch.randint(W, (B,), generator=g)
    cfg = _atlas_cfg(tr, B, False)
    nbytes = int(tr.lib.b200_atlas_workspace_bytes_for(C.byref(cfg), C.byref(tr.map_desc)))
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
    ysd, xsd = ys.to(DEV), xs.to(DEV)
    N.check(tr.lib.b200_pretrain_loss_grad_for(C.byref(cfg), C.byref(tr.map_desc), larger, T, f, N.ptr(ysd), N.ptr(xsd),
                                               N.ptr(tr.params), N.ptr(tr.grads), N.ptr(tr.losses), N.ptr(ws),
                                               ws.numel(), N.current_stream()))
    torch.cuda.synchronize()
    v = _atlas_views(tr, cfg, ws)
    cap = v["cap"]
    hL = np.float32(larger / 2.0)
    t_norm = np.float32(f / (T / 2.0) - 1.0)
    xm = v["x_map"][0]
    ref = np.stack([_norm(xs.numpy().astype(np.float32), hL), _norm(ys.numpy().astype(np.float32), hL),
                    np.full(B, t_norm, np.float32), np.zeros(B, np.float32)], axis=1)
    assert np.array_equal(xm[:B].view(np.uint32), ref.view(np.uint32))
    assert np.all(xm[B:cap] == 0) and int(v["counters"][0]) == B
    rt = Ratios(f"pretrain B={B} {'tc' if prec else 'fp32'}")
    s = f32(cfg.uv_mapping_scale)
    u = vec(v["uv"][0, :B])
    ex, ey = E(xm[:B, 0]) * s - u[0], E(xm[:B, 1]) * s - u[1]
    ns = ex * ex + ey * ey
    n = ns.sqrt()
    assert not ns.undecided().any()
    inv = 1.0 / n
    ib = inv_of(B)
    rt.close("d_uv0", v["d_uv"][0, :B, 0], -ib * ex * inv)
    rt.close("d_uv1", v["d_uv"][0, :B, 1], -ib * ey * inv)
    assert np.all(v["d_uv"][0, B:cap] == 0)
    loss = E(float(n.v.sum()), float(n.e.sum()) + (8 + cap // 32) * float(n.v.sum())) * ib
    rt.close("loss", tr.losses.cpu().numpy()[0], loss)
    assert np.all(np.isfinite(tr.grads.cpu().numpy()))
    assert rt.report() <= 1.0


# ------------------------------------------------------------------------------------------------ (d) segmentation trip
def seg_head(uv1, uv2, ar, y, tg, wf, wb, cfg, larger, B, n_f, n_b):
    """seg_sample_loss of seg_loss_math.h in float64 (alpha from the exact fp32 seg_alpha)."""
    n = tg.shape[0]
    und = np.zeros(n, bool)
    f = np.float32
    a_ = [(((f(0.5) * (ar[k].astype(f) + f(1.0))).astype(f) * f(0.99)).astype(f) + f(0.001)).astype(f)
          for k in range(5)]
    a = [E(x.astype(np.float64)) for x in a_]
    da = [E(np.zeros(n)) for _ in range(5)]
    al, ax, ay = a[0], a[1], a[2]
    ib = inv_of(B)
    w_rgb, w_grad, w_sp = (E(f32(c)) * ib for c in (cfg.rgb_coeff, cfg.gradient_coeff, cfg.sparsity_coeff))
    dy = [[None] * 3 for _ in range(6)]
    val = {k: E(np.zeros(n)) for k in ("rgb", "grad", "sp")}
    for ch in range(3):
        c = [(E(y[k][:, ch]) + 1.0) * 0.5 for k in range(6)]
        o = c[0] * al + c[3] * (1.0 - al)
        ox = c[1] * ax + c[4] * (1.0 - ax)
        oy = c[2] * ay + c[5] * (1.0 - ay)
        nn_ = c[0] * (1.0 - al)
        e = o - E(tg[:, ch])
        ex, ey = E(tg[:, 3 + ch]) - (ox - o), E(tg[:, 6 + ch]) - (oy - o)
        val["rgb"] = val["rgb"] + e * e
        val["grad"] = val["grad"] + (ex * ex + ey * ey)
        val["sp"] = val["sp"] + nn_ * nn_
        g_o = w_rgb * 2.0 * e + w_grad * 2.0 * (ex + ey)
        g_ox, g_oy, g_n = -w_grad * 2.0 * ex, -w_grad * 2.0 * ey, w_sp * 2.0 * nn_
        dy[0][ch] = 0.5 * (g_o * al + g_n * (1.0 - al)); dy[3][ch] = 0.5 * (g_o * (1.0 - al))
        dy[1][ch] = 0.5 * (g_ox * ax); dy[4][ch] = 0.5 * (g_ox * (1.0 - ax))
        dy[2][ch] = 0.5 * (g_oy * ay); dy[5][ch] = 0.5 * (g_oy * (1.0 - ay))
        da[0] = da[0] + (g_o * (c[0] - c[3]) - g_n * c[0])
        da[1] = da[1] + g_ox * (c[1] - c[4])
        da[2] = da[2] + g_oy * (c[2] - c[5])
    L, s = float(larger), f32(cfg.uv_mapping_scale)
    d1 = [[E(np.zeros(n)), E(np.zeros(n))] for _ in range(9)]
    d2 = [[E(np.zeros(n)), E(np.zeros(n))] for _ in range(9)]
    U1, U2 = [vec(uv1[g]) for g in range(9)], [vec(uv2[g]) for g in range(9)]
    cr = E(f32(cfg.rigidity_coeff)) * ib
    val["r1"] = rigidity(U1[0], U1[3], U1[4], L, s, f32(cfg.derivative_amount), cr, d1[0], d1[3], d1[4], und)
    val["r2"] = rigidity(U2[0], U2[3], U2[4], L, s, f32(cfg.derivative_amount), cr, d2[0], d2[3], d2[4], und)
    val["g1"] = val["g2"] = E(np.zeros(n))
    if cfg.with_global:
        dg = f32(cfg.global_derivative_amount)
        val["g1"] = rigidity(U1[0], U1[7], U1[8], L, s, dg, E(f32(cfg.global_rigidity_coeff_fg)) * ib, d1[0], d1[7],
                             d1[8], und)
        val["g2"] = rigidity(U2[0], U2[7], U2[8], L, s, dg, E(f32(cfg.global_rigidity_coeff_bg)) * ib, d2[0], d2[7],
                             d2[8], und)
    for dr, (on, g, ak, cntn) in enumerate(((wf, G_FWD, 3, n_f), (wb, G_BWD, 4, n_b))):
        inv_n = inv_of(cntn)
        wm = E(0.5 * f32(cfg.flow_coeff)) * inv_n
        l1 = flow(U1[0], U1[g], L, s, wm * al, d1[0], d1[g], und, on)
        l2 = flow(U2[0], U2[g], L, s, wm * (1.0 - al), d2[0], d2[g], und, on)
        val[f"f1{dr}"], val[f"f2{dr}"] = where(on, l1 * al, 0.0), where(on, l2 * (1.0 - al), 0.0)
        da[0] = where(on, da[0] + wm * (l1 - l2), da[0])
        dd = (a_[0] - a_[ak]) if dr == 0 else (a_[ak] - a_[0])          # exact fp32 difference: its sign is exact
        sg = np.sign(dd).astype(np.float64)
        wa = E(0.5 * f32(cfg.alpha_flow_factor)) * inv_n * E(sg)
        val[f"a{dr}"] = where(on, E(np.abs(dd).astype(np.float64)), 0.0)
        if dr == 0:
            da[0] = where(on, da[0] + wa, da[0]); da[ak] = where(on, da[ak] - wa, da[ak])
        else:
            da[ak] = where(on, da[ak] + wa, da[ak]); da[0] = where(on, da[0] - wa, da[0])
    agt = E(tg[:, 11])
    val["bce"] = -agt * al.log() - (1.0 - agt) * (1.0 - al).log()
    da[0] = da[0] + E(f32(cfg.bootstrapping_factor)) * ib * (-agt / al + (1.0 - agt) / (1.0 - al))
    dar = [E(f32(0.495)) * x for x in da]
    return d1, d2, dar, dy, val, und


@pytest.mark.parametrize("prec", [N.PREC_FP32, N.PREC_TC], ids=["fp32", "tc"])
@pytest.mark.parametrize("world", [1, 2])
def test_seg_trip_glue_and_head(golden_dir, prec, world):
    if prec == N.PREC_TC and not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")
    z, video, masks, _ = load_fixture(golden_dir)
    data = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("video_")}
    inds = torch.from_numpy(z["inds"])
    B = inds.shape[0]
    H, W, _, T = data["frames"].shape
    for r in range(world):
        t0, t1 = A.frame_range(r, world, T) if world > 1 else (0, T)
        vid = A.DeviceVideo.from_reference_layout(data, DEV, t0, t1)
        tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, DEV, t0, t1), {"samples_batch": B}, precision=prec, device=DEV)
        torch.manual_seed(int(z["init_seed"]))
        tr.init_like_reference()
        cfg = tr._config(0)
        nbytes = int(tr.lib.b200_seg_workspace_bytes(C.byref(cfg)))
        ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
        idx = inds.reshape(-1).to(DEV)
        N.check(tr.lib.b200_seg_loss_grad(C.byref(cfg), C.byref(vid.struct), N.ptr(tr.mask), N.ptr(idx), N.ptr(tr.params),
                                          N.ptr(tr.grads), N.ptr(tr.losses), N.ptr(ws), ws.numel(), N.current_stream()))
        torch.cuda.synchronize()
        off = (C.c_int64 * N.SEG_OFFSET_FLOATS)()
        N.check(tr.lib.b200_seg_workspace_offsets(C.byref(cfg), N.ptr(ws), off))
        cap = (B + 127) // 128 * 128

        def fv(i, *shape):
            n = int(np.prod(shape))
            return ws[off[i]:off[i] + 4 * n].view(torch.float32).cpu().numpy().reshape(shape)
        cnt = ws[off[0]:off[0] + 32].view(torch.int32).cpu().numpy()
        xm, tg, x3, xa, xat = fv(1, 9, cap, 4), fv(2, cap, 12), fv(3, 9, cap, 3), fv(4, 5, cap, 3), fv(5, 6, cap, 2)
        uv1, uv2, ar, yat = fv(6, 9, cap, 2), fv(7, 9, cap, 2), fv(8, 5, cap), fv(9, 6, cap, 3)
        d_uv1, d_uv2, d_ar, d_yat, d_xat = fv(10, 9, cap, 2), fv(11, 9, cap, 2), fv(12, 5, cap), fv(13, 6, cap, 3), \
            fv(14, 6, cap, 2)
        # sampling, with the matte of each sample in target column 11
        t, y, x, _ = _records(data, inds)
        matte = masks.numpy()[y, x, t].astype(np.float32)
        v = dict(cap=cap, counters=cnt, x_map=xm, targets=tg)
        pf, pb = check_sampling(v, data, inds, cfg, 9, t0, t1, matte)
        n_local, n_f, n_b = int(cnt[0]), int(cnt[1]), int(cnt[2])
        # glue, bit for bit
        assert np.array_equal(x3.view(np.uint32), xm[:, :, :3].view(np.uint32))
        for k, g in enumerate((0, 1, 2, G_FWD, G_BWD)):
            assert np.array_equal(xa[k].view(np.uint32), xm[g, :, :3].view(np.uint32)), f"alpha row group {k}"
        h = np.float32(0.5)
        live = np.isfinite(uv1[:3]).all(-1) & np.isfinite(uv2[:3]).all(-1)       # rows the networks evaluated
        assert live[:, :n_local].all()
        assert np.array_equal(xat[:3][live].view(np.uint32), (uv1[:3][live] * h + h).astype(np.float32).view(np.uint32))
        assert np.array_equal(xat[3:][live].view(np.uint32), (uv2[:3][live] * h - h).astype(np.float32).view(np.uint32))
        # loss head
        s = np.arange(n_local)
        rows = [np.maximum(pf, 0) if g == G_FWD else (np.maximum(pb, 0) if g == G_BWD else s) for g in range(9)]
        pick = lambda a, g: np.where(((g != G_FWD) | (pf >= 0)) & ((g != G_BWD) | (pb >= 0)), a[g, rows[g]].T, 0).T
        u1, u2 = np.stack([pick(uv1, g) for g in range(9)]), np.stack([pick(uv2, g) for g in range(9)])
        arr = [np.where(((k != 3) | (pf >= 0)) & ((k != 4) | (pb >= 0)),
                        ar[k, rows[(0, 1, 2, G_FWD, G_BWD)[k]]], 0) for k in range(5)]
        d1, d2, dar, dy, val, und = seg_head(u1, u2, arr, yat[:, :n_local], tg[:n_local], pf >= 0, pb >= 0, cfg,
                                             max(H, W), B, n_f, n_b)
        assert not und.any()
        rt = Ratios(f"seg {'tc' if prec else 'fp32'} shard {r}/{world}")
        for k in range(6):
            for c in range(3):
                rt.close(f"d_yat{k}", d_yat[k, :n_local, c], dy[k][c])
        for k in range(5):
            if k >= 3:
                p = pf if k == 3 else pb
                sel = p >= 0
                rt.close(f"d_ar{k}", d_ar[k, p[sel]], E(dar[k].v[sel], dar[k].e[sel]))
            else:
                rt.close(f"d_ar{k}", d_ar[k, :n_local], dar[k])
        for name, dd, dev in (("d_uv1", d1, d_uv1), ("d_uv2", d2, d_uv2)):
            for g in range(9):
                for c in range(2):
                    if g in (G_FWD, G_BWD):
                        p = pf if g == G_FWD else pb
                        sel = p >= 0
                        rt.close(f"{name}.{g}", dev[g, p[sel], c], E(dd[g][c].v[sel], dd[g][c].e[sel]))
                    elif g >= 3:
                        rt.close(f"{name}.{g}", dev[g, :n_local, c], dd[g][c])
                    else:
                        # seg_chain_kernel: final = fl(head + 0.5 d_xat); one ulp of final on top of the head's bound
                        layer = 0 if name == "d_uv1" else 3
                        fin = dev[g, :n_local, c]
                        half = 0.5 * d_xat[layer + g, :n_local, c].astype(np.float64)
                        ulp = np.spacing(np.abs(fin)).astype(np.float64)
                        ref = E(dd[g][c].v, dd[g][c].e + ulp / (C_ENV * U))
                        rt.close(f"{name}.{g}chain", fin.astype(np.float64) - half, ref)
        assert np.all(d_uv1[:3, n_local:] == 0) and np.all(d_uv2[:3, n_local:] == 0)
        assert np.all(d_yat[:, n_local:] == 0)
        # the 14-float loss vector
        losses = tr.losses.cpu().numpy()
        nb = (cap + 127) // 128
        ib = inv_of(B)
        bs = lambda k, sc=ib: block_sum(val[k], sc, nb)
        ref = {1: bs("rgb"), 2: bs("grad"), 3: bs("sp"), 4: bs("r1"), 5: bs("r2"), 6: bs("g1"), 7: bs("g2"),
               11: bs("bce")}
        for i, k in ((8, "f1"), (9, "f2"), (10, "a")):
            ref[i] = 0.5 * (block_sum(val[f"{k}0"], inv_of(n_f), nb) + block_sum(val[f"{k}1"], inv_of(n_b), nb))
        for i, e in ref.items():
            rt.close(f"loss{i}", losses[i], e)
        assert losses[12] == n_f and losses[13] == n_b
        tot = (E(f32(cfg.rigidity_coeff)) * (ref[4] + ref[5]) + E(f32(cfg.global_rigidity_coeff_fg)) * ref[6]
               + E(f32(cfg.global_rigidity_coeff_bg)) * ref[7] + E(f32(cfg.rgb_coeff)) * ref[1]
               + E(f32(cfg.flow_coeff)) * (ref[8] + ref[9]) + E(f32(cfg.bootstrapping_factor)) * ref[11]
               + E(f32(cfg.alpha_flow_factor)) * ref[10] + E(f32(cfg.sparsity_coeff)) * ref[3]
               + E(f32(cfg.gradient_coeff)) * ref[2])
        rt.close("loss0", losses[0], E(tot.v, tot.e + nb * abs(tot.v)))
        assert np.all(np.isfinite(tr.grads.cpu().numpy()))
        assert rt.report() <= 1.0
        del ws, tr, vid


# ------------------------------------------------------------------------------------------------ (e) stand-alone heads
HEAD_SIZES = [1, 31, 32, 127, 128, 129, (1 << 20) + 3]


def _head_inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    uv = torch.rand(n, 2, generator=g) * 2 - 1
    nb = uv.repeat(2, 1) + 0.05 * torch.randn(2 * n, 2, generator=g)
    m = uv + 0.05 * torch.randn(n, 2, generator=g)
    # exact edges on a few rows: identical neighbours (A = B = D = 0), identical flow match (n = 0)
    k = max(1, n // 7)
    nb[:k] = uv[:k]
    nb[n:n + k] = uv[:k]
    m[-k:] = uv[-k:]
    w = torch.rand(n, generator=g)
    w[:k] = 0.0
    w[k:2 * k] = 1.0
    return uv, nb, m, w, k


@pytest.mark.parametrize("n", HEAD_SIZES)
def test_standalone_heads(n):
    lib, st = N.lib(), N.current_stream()
    uv, nb, m, w, k = _head_inputs(n, n)
    L, s, d = 40.0, f32(0.8), 1.0
    rt = Ratios(f"heads n={n}")
    inv_n = inv_of(n)
    nblk = (n + 127) // 128
    dv = lambda t: t.to(DEV).contiguous()
    uv_d, nb_d, m_d, w_d = dv(uv), dv(nb), dv(m), dv(w)
    # gradient head
    g = torch.Generator().manual_seed(n + 1)
    rgb, xp, yp, dxg, dyg = (torch.rand(n, 3, generator=g) for _ in range(5))
    loss = torch.zeros(1, device=DEV)
    outs = [torch.empty(n, 3, device=DEV) for _ in range(3)]
    ins = [dv(t) for t in (rgb, xp, yp, dxg, dyg)]             # kept alive until the kernels have run
    N.check(lib.b200_gradient_loss_head(*(N.ptr(t) for t in ins), n, N.ptr(loss), *(N.ptr(o) for o in outs), st))
    torch.cuda.synchronize()
    part = E(np.zeros(n))
    for c in range(3):
        o = E(rgb[:, c].double().numpy())
        ex = E(dxg[:, c].double().numpy()) - (E(xp[:, c].double().numpy()) - o)
        ey = E(dyg[:, c].double().numpy()) - (E(yp[:, c].double().numpy()) - o)
        part = part + (ex * ex + ey * ey)
        rt.close("grad.d_rgb", outs[0][:, c].cpu().numpy(), 2.0 * (ex + ey) * inv_n)
        rt.close("grad.d_xp", outs[1][:, c].cpu().numpy(), -2.0 * ex * inv_n)
        rt.close("grad.d_yp", outs[2][:, c].cpu().numpy(), -2.0 * ey * inv_n)
    rt.close("grad.loss", loss.cpu().numpy()[0], block_sum(part, inv_n, nblk))
    # rigidity head, with and without the per-sample output
    for with_ps in (False, True):
        ps = torch.full((n,), -7.0, device=DEV) if with_ps else None
        d_uv, d_uvp = torch.empty(n, 2, device=DEV), torch.empty(2 * n, 2, device=DEV)
        N.check(lib.b200_rigidity_loss_head(N.ptr(uv_d), N.ptr(nb_d), n, L, s, d, N.ptr(ps), N.ptr(loss),
                                            N.ptr(d_uv), N.ptr(d_uvp), st))
        torch.cuda.synchronize()
        g0 = [E(np.zeros(n)), E(np.zeros(n))]
        ga, gb = [E(np.zeros(n)), E(np.zeros(n))], [E(np.zeros(n)), E(np.zeros(n))]
        und = np.zeros(n, bool)
        u0, nbn = vec(uv.numpy()), nb.numpy()
        val = rigidity(u0, vec(nbn[:n]), vec(nbn[n:]), L, s, d, inv_n, g0, ga, gb, und)
        assert not und.any()
        for c in range(2):
            rt.close("rig.d_uv", d_uv[:, c].cpu().numpy(), g0[c])
            rt.close("rig.d_uva", d_uvp[:n, c].cpu().numpy(), ga[c])
            rt.close("rig.d_uvb", d_uvp[n:, c].cpu().numpy(), gb[c])
        if with_ps:
            rt.close("rig.per_sample", ps.cpu().numpy(), val)
        rt.close("rig.loss", loss.cpu().numpy()[0], block_sum(val, inv_n, nblk))
    # flow heads, plain and weighted
    for weighted in (False, True):
        d_rel, d_m = torch.empty(n, 2, device=DEV), torch.empty(n, 2, device=DEV)
        d_w = torch.empty(n, device=DEV)
        if weighted:
            N.check(lib.b200_flow_loss_head_weighted(N.ptr(uv_d), N.ptr(m_d), N.ptr(w_d), n, L, s, N.ptr(loss),
                                                     N.ptr(d_rel), N.ptr(d_m), N.ptr(d_w), st))
        else:
            N.check(lib.b200_flow_loss_head(N.ptr(uv_d), N.ptr(m_d), n, L, s, N.ptr(loss), N.ptr(d_rel), N.ptr(d_m),
                                            st))
        torch.cuda.synchronize()
        wE = E(w.double().numpy()) if weighted else None
        coeff = inv_n * wE if weighted else inv_n
        g0, gm = [E(np.zeros(n)), E(np.zeros(n))], [E(np.zeros(n)), E(np.zeros(n))]
        und = np.zeros(n, bool)
        lv = flow(vec(uv.numpy()), vec(m.numpy()), L, s, coeff, g0, gm, und)
        assert not und.any()
        tag = "wflow" if weighted else "flow"
        for c in range(2):
            rt.close(f"{tag}.d_rel", d_rel[:, c].cpu().numpy(), g0[c])
            rt.close(f"{tag}.d_match", d_m[:, c].cpu().numpy(), gm[c])
        # identical match: value 0 and gradient exactly 0; w = 0: gradient exactly 0
        assert torch.all(d_rel[-k:] == 0) and torch.all(d_m[-k:] == 0)
        if weighted:
            assert torch.all(d_rel[:k] == 0) and torch.all(d_m[:k] == 0)
            rt.close("wflow.d_w", d_w.cpu().numpy(), lv * inv_n)
            rt.close("wflow.loss", loss.cpu().numpy()[0], block_sum(lv * wE, inv_n, nblk))
        else:
            rt.close("flow.loss", loss.cpu().numpy()[0], block_sum(lv, inv_n, nblk))
    assert rt.report() <= 1.0


def test_flow_heads_on_empty_sets():
    """n = 0: the loss is the NaN of a mean over nothing, and no gradient buffer is touched."""
    lib, st = N.lib(), N.current_stream()
    loss = torch.zeros(1, device=DEV)
    bufs = [torch.full((8,), 3.5, device=DEV) for _ in range(3)]
    N.check(lib.b200_flow_loss_head(N.ptr(bufs[0]), N.ptr(bufs[0]), 0, 40.0, 0.8, N.ptr(loss), N.ptr(bufs[1]),
                                    N.ptr(bufs[2]), st))
    torch.cuda.synchronize()
    assert torch.isnan(loss).all() and all(torch.all(b == 3.5) for b in bufs)
    loss.zero_()
    w = torch.full((8,), 3.5, device=DEV)
    N.check(lib.b200_flow_loss_head_weighted(N.ptr(bufs[0]), N.ptr(bufs[0]), N.ptr(w), 0, 40.0, 0.8, N.ptr(loss),
                                             N.ptr(bufs[1]), N.ptr(bufs[2]), N.ptr(w), st))
    torch.cuda.synchronize()
    assert torch.isnan(loss).all() and all(torch.all(b == 3.5) for b in bufs) and torch.all(w == 3.5)


# ------------------------------------------------------------------------------------------------ (f) workspace fill
def _agree(name, a, b, n_params, tol):
    la, lb = a[n_params:], b[n_params:]
    ga, gb = a[:n_params], b[:n_params]
    assert torch.all(torch.isfinite(ga)) and torch.all(torch.isfinite(gb)), f"{name}: non-finite gradients"
    assert torch.all(torch.isfinite(la[:6])) and torch.all(torch.isfinite(lb[:6])), f"{name}: non-finite losses"
    np.testing.assert_allclose(la.cpu().numpy(), lb.cpu().numpy(), rtol=1e-5)
    assert (ga - gb).norm() <= tol * gb.norm(), name


@pytest.mark.parametrize("prec", [N.PREC_FP32, N.PREC_TC], ids=["fp32", "tc"])
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("with_global", [True, False], ids=["global", "local"])
def test_atlas_step_ignores_workspace_contents(golden_dir, prec, world, with_global):
    """A step on a workspace of 0xFF bytes (NaN as fp32) gives what it gives on a zeroed one."""
    if prec == N.PREC_TC and not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")
    data, inds = _golden_video(golden_dir)
    B, T = inds.shape[0], data["frames"].shape[3]
    for r in range(world):
        t0, t1 = A.frame_range(r, world, T) if world > 1 else (0, T)
        tr = _atlas_trainer(data, golden_dir, B, prec, 0, t0, t1)
        cfg = _atlas_cfg(tr, B, with_global)
        out = []
        for fill in (0xFF, 0):
            _atlas_step(tr, cfg, inds, fill)
            out.append(tr.grad_loss.clone())
        _agree(f"atlas shard {r}/{world}", out[0], out[1], tr.n_params, 1e-4)


@pytest.mark.parametrize("prec", [N.PREC_FP32, N.PREC_TC], ids=["fp32", "tc"])
def test_seg_and_pretrain_ignore_workspace_contents(golden_dir, prec):
    if prec == N.PREC_TC and not N.lib().b200_device_supports_tc():
        pytest.skip("needs sm_90")
    z, video, masks, _ = load_fixture(golden_dir)
    data = {k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("video_")}
    inds = torch.from_numpy(z["inds"]).reshape(-1).to(DEV)
    vid = A.DeviceVideo.from_reference_layout(data, DEV)
    tr = SG.SegTrainer(vid, SG.pack_mask_frames(masks, DEV), {"samples_batch": inds.numel()}, precision=prec, device=DEV)
    torch.manual_seed(int(z["init_seed"]))
    tr.init_like_reference()
    cfg = tr._config(0)
    nbytes = int(tr.lib.b200_seg_workspace_bytes(C.byref(cfg)))
    out = []
    for fill in (0xFF, 0):
        ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=DEV)
        N.check(tr.lib.b200_seg_loss_grad(C.byref(cfg), C.byref(vid.struct), N.ptr(tr.mask), N.ptr(inds), N.ptr(tr.params),
                                          N.ptr(tr.grads), N.ptr(tr.losses), N.ptr(ws), ws.numel(), N.current_stream()))
        torch.cuda.synchronize()
        out.append(tr.grad_loss.clone())
    _agree("seg", out[0], out[1], tr.n_params, 1e-4)
    # pre-training of the atlas step's mapping on the same kind of workspace
    atr = _atlas_trainer(data, golden_dir, 64, prec, 0)
    B = 1000
    g = torch.Generator().manual_seed(2)
    ys, xs = torch.randint(24, (B,), generator=g).to(DEV), torch.randint(40, (B,), generator=g).to(DEV)
    acfg = _atlas_cfg(atr, B, False)
    nbytes = int(atr.lib.b200_atlas_workspace_bytes_for(C.byref(acfg), C.byref(atr.map_desc)))
    out = []
    for fill in (0xFF, 0):
        ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=DEV)
        N.check(atr.lib.b200_pretrain_loss_grad_for(C.byref(acfg), C.byref(atr.map_desc), 40, 6, 2, N.ptr(ys), N.ptr(xs),
                                                    N.ptr(atr.params), N.ptr(atr.grads), N.ptr(atr.losses), N.ptr(ws),
                                                    ws.numel(), N.current_stream()))
        torch.cuda.synchronize()
        out.append(atr.grad_loss.clone())
    n = atr.map_total
    assert torch.all(torch.isfinite(out[0][:n])) and np.isfinite(out[0][atr.n_params].item())
    np.testing.assert_allclose(out[0][atr.n_params].item(), out[1][atr.n_params].item(), rtol=1e-5)
    assert (out[0][:n] - out[1][:n]).norm() <= 1e-4 * out[1][:n].norm()
