"""Adam (adam_kernel, b200_adam_step) and the fused data-parallel step (dp_adam_kernel, b200_dp_adam_step) against
float64 on the kernels' own operands, and the exchange bit for bit with 1 to 16 ranks emulated on one GPU.

Float64 restatement.  Before every step the test reads p, m, v and the step counter t back from the device and
restates the step in float64, in the order the kernel computes it:
  w1 = fp32(1 - b1), w2 = fp32(1 - b2), b2 and eps as fp32;  step_size = lr / (1 - b1^t), bc2_sqrt = sqrt(1 - b2^t)
  m' = m + w1 (g - m);  v' = v b2 + (w2 g) g;  denom = sqrt(v') / bc2_sqrt + eps;  p' = p + (-step_size m') / denom
Every operation carries a first-order running-error envelope (the scheme of test_stage1_heads_gpu.py): it adds one
rounding of its result, max(|result|, 2^-126) in units of u = 2^-24, so that the absolute error 2^-150 of a subnormal
result is covered, and the envelopes of its operands propagate through the absolute partial derivatives.  step_size
and bc2_sqrt enter with one rounding each, because the device rounds them to fp32 from its own pow.  sqrt propagates
|sqrt(a) - sqrt(b)| <= min(|a - b| / sqrt(a), sqrt(|a - b|)), which also holds where v' is subnormal.  A device value
must lie within  C_ENV * u * envelope + 2^-149  of the float64 value.  Restating each step on the kernel's own state
keeps errors from compounding, so the bound does not depend on the number of steps.  Each case prints its largest
ratio of error to bound.

Emulated ranks.  dp_adam_kernel waits on flag words that other ranks publish.  Here the ranks' launches run one after
another on one stream, each followed by a synchronisation, so no two exchange kernels ever run at the same time and
the device-wide ticket of the kernel is never shared.  Before rank R launches, the test presets to the current epoch
only the flag words no other rank can have written yet (those of the ranks that have not run in this step, and R's
own two), reads back all 2W words R awaits and fails without launching unless every one is >= the epoch.  So no
launch can wait on a flag, and the check shows that every rank that ran earlier published both rounds to R.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from b200 import _native as N
from b200 import atlas as A
from b200 import seg as SG

DEV = "cuda"
U = 2.0 ** -24
C_ENV = 4.0
TINY = 2.0 ** -126          # smallest normal: a rounding's absolute error is at most u * max(|result|, TINY)
FLOOR = 2.0 ** -149         # smallest subnormal: floor of every bound
LR, B1, B2, EPS = 1e-4, 0.9, 0.999, 1e-8
SENTINEL = 1234.5
SHIPPED_STEPS = 9999        # the counter before the last step of the shipped 10 000-iteration loop
MULTIWAVE_BLOCKS = 2048     # adam_kernel blocks (1024 floats each) of the multi-wave sizes; more than an H100 holds


# ------------------------------------------------------------------------------------------------ float64 + envelope
class E:
    """float64 value with a first-order running-error envelope (in units of u)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v, self.e = np.broadcast_arrays(np.asarray(v, dtype=np.float64), np.asarray(e, dtype=np.float64))

    @staticmethod
    def w(x):
        return x if isinstance(x, E) else E(x)

    @staticmethod
    def rnd(v):
        return np.maximum(np.abs(v), TINY)

    def __add__(self, o):
        o = E.w(o); v = self.v + o.v
        return E(v, self.e + o.e + E.rnd(v))

    __radd__ = __add__

    def __sub__(self, o):
        o = E.w(o); v = self.v - o.v
        return E(v, self.e + o.e + E.rnd(v))

    def __mul__(self, o):
        o = E.w(o); v = self.v * o.v
        return E(v, np.abs(o.v) * self.e + np.abs(self.v) * o.e + E.rnd(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = E.w(o); v = self.v / o.v
        return E(v, self.e / np.abs(o.v) + np.abs(self.v) * o.e / (o.v * o.v) + E.rnd(v))

    def __neg__(self):
        return E(-self.v, self.e)

    def sqrt(self):
        v = np.sqrt(self.v)
        d = C_ENV * U * self.e                                  # bound on the operand's absolute error
        with np.errstate(divide="ignore", invalid="ignore"):
            lin = np.where(v > 0, d / np.where(v > 0, v, 1.0), np.inf)
        return E(v, np.minimum(lin, np.sqrt(d)) / (C_ENV * U) + E.rnd(v))

    def bound(self):
        return C_ENV * U * self.e + FLOOR


def adam_f64(p, m, v, g, t, grad_scale=1.0):
    """One step of adam_kernel on fp32 operands, restated in float64 with envelopes: (p', m', v')."""
    w1, w2, b2, eps = (float(np.float32(x)) for x in (1.0 - B1, 1.0 - B2, B2, EPS))
    ss, bc = LR / (1.0 - B1 ** t), np.sqrt(1.0 - B2 ** t)
    step_size, bc2_sqrt = E(ss, ss), E(bc, bc)
    gs = float(np.float32(grad_scale))
    ga = E(g) if gs == 1.0 else E(g) * gs
    m0, v0 = E(m), E(v)
    m1 = m0 + w1 * (ga - m0)
    v1 = v0 * b2 + (w2 * ga) * ga
    denom = v1.sqrt() / bc2_sqrt + eps
    p1 = E(p) + (-step_size * m1) / denom
    return p1, m1, v1


class Worst:
    """The checks against the envelope, and the largest ratio of error to bound per quantity."""

    def __init__(self, case):
        self.case, self.r = case, {}

    def check(self, what, got, ref):
        got = np.asarray(got, dtype=np.float64)
        assert np.all(np.isfinite(ref.v)), (self.case, what, "non-finite float64 value")
        assert np.all(np.isfinite(got)), (self.case, what, "non-finite device value")
        err, bnd = np.abs(got - ref.v), ref.bound()
        bad = ~(err <= bnd)
        if bad.any():
            i = int(np.argmax(bad))
            raise AssertionError(f"{self.case} {what}: {int(bad.sum())} entries out of bound, first at {i}: device "
                                 f"{got[i]!r} float64 {ref.v[i]!r} bound {bnd[i]!r}")
        self.r[what] = max(self.r.get(what, 0.0), float((err / bnd).max()))

    def step(self, p, m, v, ref):
        for what, got, r in zip("pmv", (p, m, v), ref):
            self.check(what, got, r)

    def report(self):
        print(f"{self.case}: largest error/bound " + ", ".join(f"{k} {x:.3f}" for k, x in sorted(self.r.items())))


def host(t):
    return t.detach().cpu().numpy().copy()


def same(a, b):
    """Bit-identical fp32 tensors."""
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def all_sentinel(t):
    return bool((t.view(torch.int32) == int(np.float32(SENTINEL).view(np.int32))).all())


# ------------------------------------------------------------------------------------------------ sizes
@functools.lru_cache(None)
def _trainer_sizes():
    """n_params of both stage-1 variants."""
    return (A.AtlasTrainer(None, device="cpu").n_params, SG.SegTrainer(None, None, device="cpu").n_params)


def _adam_size(name):
    if isinstance(name, int):
        return name
    if name == "atlas":
        return int(N.lib().b200_atlas_param_floats())
    if name == "seg":
        return _trainer_sizes()[1]
    return 1024 * MULTIWAVE_BLOCKS + (1 if name.endswith("+1") else -1)


def _spread(rng, n, zero):
    """fp32 values of random sign with magnitudes log-uniform over 1e-22 .. 1e18, both ends present; 0 where `zero`.
    At the small end g^2 underflows to a subnormal or to 0; at the large end (w2 g) g ~ 1e33 stays finite."""
    mag = 10.0 ** rng.uniform(-22.0, 18.0, n)
    mag[0] = 1e-22
    if n > 1:
        mag[-1] = 1e18
    g = (mag * rng.choice([-1.0, 1.0], n)).astype(np.float32)
    g[zero] = 0.0
    return g


def _zero_mask(rng, n):
    """Entries with g = m = v = 0 at every step: v' = 0 and denom = eps."""
    zero = rng.random(n) < 1.0 / 16
    zero[0] = zero[-1] = False
    if n >= 3:
        zero[1] = True
    return zero


def _moments(rng, g, zero):
    """Non-zero starting moments on the scale of the gradients (v underflows where g does)."""
    m = (g.astype(np.float64) * rng.standard_normal(g.size)).astype(np.float32)
    v = ((g.astype(np.float64) * rng.uniform(0.0, 2.0, g.size)) ** 2).astype(np.float32)
    m[zero] = 0.0
    v[zero] = 0.0
    return m, v


def _adam(p, g, m, v, n, step, grad_scale=1.0):
    N.check(N.lib().b200_adam_step(N.ptr(p), N.ptr(g), N.ptr(m), N.ptr(v), n, LR, B1, B2, EPS, grad_scale, N.ptr(step),
                                   N.current_stream()), "b200_adam_step")


# ------------------------------------------------------------------------------------------------ b200_adam_step
ADAM_SIZES = [1, 2, 3, 4, 5, 255, 1021, 1024, 1025, "multiwave-1", "multiwave+1", "atlas", "seg"]


@pytest.mark.gpu
@pytest.mark.parametrize("grad_scale", [1.0, 0.5, 1.0 / 3.0])
@pytest.mark.parametrize("size", ADAM_SIZES)
def test_adam_step_against_float64(size, grad_scale):
    """Steps t = 1, 2, 3 and a step from the counter preset to 9 999, where 1 - b1^t is 1 in float64 and only the
    second bias correction is left.  Sizes: the scalar tail (n mod 4 = 1, 2, 3), one block and one float past it,
    grids larger than the device holds at once (the counter then advances through the last block's ticket) and both
    stage-1 parameter buffers.  The counter advances by exactly one per call."""
    n = _adam_size(size)
    if not isinstance(size, int) and size.startswith("multiwave"):
        pr = torch.cuda.get_device_properties(0)
        assert MULTIWAVE_BLOCKS * 256 > pr.multi_processor_count * pr.max_threads_per_multi_processor
    rng = np.random.default_rng([n, round(grad_scale * 1000)])
    zero = _zero_mask(rng, n)
    m0, v0 = _moments(rng, _spread(rng, n, zero), zero)
    p = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(DEV)
    m, v = torch.from_numpy(m0).to(DEV), torch.from_numpy(v0).to(DEV)
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    worst = Worst(f"adam n={n} grad_scale={grad_scale:.4g}")
    for preset in (None, None, None, SHIPPED_STEPS):
        if preset is not None:
            step.fill_(preset)
        g = _spread(rng, n, zero)
        p0, m0, v0, t0 = host(p), host(m), host(v), int(step)
        _adam(p, torch.from_numpy(g).to(DEV), m, v, n, step, grad_scale)
        torch.cuda.synchronize()
        assert int(step) == t0 + 1, (n, t0, int(step))
        worst.step(host(p), host(m), host(v), adam_f64(p0, m0, v0, g, t0 + 1, grad_scale))
    worst.report()


@pytest.mark.gpu
@pytest.mark.parametrize("variant,which", [("atlas", "mapping"), ("seg", "mapping1"), ("seg", "mapping2"),
                                           ("seg", "alpha")])
def test_pretrain_slice_adam_against_float64(variant, which):
    """FlatTrainer.adam on one network's slice of the flat buffers at its real offset, with its own m, v and step (as
    pre-training calls it): three steps against float64, and every other float of the trainer's parameters,
    gradients, loss vector and moments keeps its sentinel; the trainer's own counter stays 0."""
    tr = A.AtlasTrainer(None, device=DEV) if variant == "atlas" else SG.SegTrainer(None, None, device=DEV)
    sl = tr.net_slice(which)
    n = sl.stop - sl.start
    for t in (tr.params, tr.grad_loss, tr.exp_avg, tr.exp_avg_sq):
        t.fill_(SENTINEL)
    rng = np.random.default_rng([n, sl.start])
    zero = _zero_mask(rng, n)
    m0, v0 = _moments(rng, _spread(rng, n, zero), zero)
    tr.params[sl] = torch.from_numpy(rng.standard_normal(n).astype(np.float32)).to(DEV)
    m, v = torch.from_numpy(m0).to(DEV), torch.from_numpy(v0).to(DEV)
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    worst = Worst(f"pretrain slice {variant}.{which} [{sl.start}, {sl.stop})")
    for _ in range(3):
        g = _spread(rng, n, zero)
        tr.grads[sl] = torch.from_numpy(g).to(DEV)
        p0, m0, v0, t0 = host(tr.params[sl]), host(m), host(v), int(step)
        tr.adam(sl, m, v, step)
        torch.cuda.synchronize()
        assert int(step) == t0 + 1
        worst.step(host(tr.params[sl]), host(m), host(v), adam_f64(p0, m0, v0, g, t0 + 1))
        assert same(tr.grads[sl], torch.from_numpy(g).to(DEV))
        for t in (tr.params, tr.grad_loss):
            assert all_sentinel(t[:sl.start]) and all_sentinel(t[sl.stop:])
        assert all_sentinel(tr.exp_avg) and all_sentinel(tr.exp_avg_sq) and int(tr.step_count) == 0
    worst.report()


@pytest.mark.gpu
def test_adam_step_counter_under_graph_replay():
    """R replays of a captured b200_adam_step on a multi-wave grid advance the counter by R and give the bytes of R
    eager calls; capturing runs nothing."""
    n, R = 1024 * MULTIWAVE_BLOCKS + 1, 5
    rng = np.random.default_rng(17)
    zero = _zero_mask(rng, n)
    g = torch.from_numpy(_spread(rng, n, zero)).to(DEV)
    m0, v0 = _moments(rng, _spread(rng, n, zero), zero)
    p0 = rng.standard_normal(n).astype(np.float32)
    eager = [torch.from_numpy(x).to(DEV) for x in (p0, m0, v0)]
    graphed = [t.clone() for t in eager]
    s_eager, s_graph = (torch.zeros(1, dtype=torch.int64, device=DEV) for _ in range(2))
    pe, me, ve = eager
    for _ in range(R):
        _adam(pe, g, me, ve, n, s_eager)
    pg, mg, vg = graphed
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _adam(pg, g, mg, vg, n, s_graph)
    torch.cuda.synchronize()
    assert int(s_graph) == 0 and same(graphed[0], torch.from_numpy(p0).to(DEV))
    for _ in range(R):
        graph.replay()
    torch.cuda.synchronize()
    assert int(s_eager) == int(s_graph) == R
    assert all(same(a, b) for a, b in zip(eager, graphed))


# ------------------------------------------------------------------------------------------------ b200_dp_adam_step
DP_WORLDS = [1, 2, 3, 4, 5, 7, 8, 16]
DP_SIZES = ["atlas", "seg", "tiny4", "tiny12"]


def _dp_size(name):
    """(n_params, n_total) of a case of the dp table."""
    atlas, seg = _trainer_sizes()
    return {"atlas": (atlas, atlas + N.LOSS_FLOATS), "seg": (seg, seg + N.SEG_LOSS_FLOATS),
            "tiny4": (4, 4 + N.LOSS_FLOATS), "tiny12": (12, 12 + N.LOSS_FLOATS)}[name]


def _dp_slice(world, rank, n_total):
    b, c = C.c_int64(), C.c_int64()
    N.check(N.lib().b200_dp_slice(world, rank, n_total, C.byref(b), C.byref(c)), "b200_dp_slice")
    return b.value, c.value


def test_dp_table_has_empty_slices_and_tail_boundaries():
    """The dp table partitions every buffer without gaps, and includes ranks whose slice is empty (total4 < W) and
    slice boundaries strictly inside the loss tail."""
    empty = inside_tail = 0
    for size in DP_SIZES:
        n_params, n_total = _dp_size(size)
        for W in DP_WORLDS:
            covered = 0
            for r in range(W):
                b, c = _dp_slice(W, r, n_total)
                assert b == covered
                covered += c
                empty += c == 0
                inside_tail += c > 0 and n_params < b < n_total
            assert covered == n_total
    assert empty > 0 and inside_tail > 0


class Ranks:
    """W emulated ranks on one device: each with its partials, parameters, moments, step, epoch and flag words, and
    the communicator that names every rank's buffers.  A rank's moments hold the sentinel outside its slice."""

    def __init__(self, W, n_params, n_total, p0, m0, v0):
        self.W, self.n_params, self.n_total = W, n_params, n_total
        self.owned = []
        for R in range(W):
            b, c = _dp_slice(W, R, n_total)
            self.owned.append(slice(min(b, n_params), min(b + c, n_params)))
        f32 = lambda: torch.zeros(n_total, dtype=torch.float32, device=DEV)
        i64 = lambda k: torch.zeros(k, dtype=torch.int64, device=DEV)
        self.partials = [f32() for _ in range(W)]
        self.params = [torch.from_numpy(p0).to(DEV) for _ in range(W)]
        self.m, self.v = [], []
        for R in range(W):
            for mine, full in ((self.m, m0), (self.v, v0)):
                t = torch.full((n_params,), SENTINEL, dtype=torch.float32, device=DEV)
                t[self.owned[R]] = torch.from_numpy(full[self.owned[R]]).to(DEV)
                mine.append(t)
        self.step, self.epoch = [i64(1) for _ in range(W)], [i64(1) for _ in range(W)]
        self.flags = [i64(2 * N.MAX_RANKS) for _ in range(W)]
        self.comm = []
        for R in range(W):
            c = N.DpComm()
            c.world, c.rank = W, R
            for j in range(W):
                c.partials[j], c.params[j] = self.partials[j].data_ptr(), self.params[j].data_ptr()
                c.flags[j] = self.flags[j].data_ptr()
            self.comm.append(c)

    def run_step(self, order, epoch):
        """One exchange step, rank after rank in `order`; a rank launches only once every flag it awaits is set."""
        W = self.W
        for k, R in enumerate(order):
            f = self.flags[R]
            for j in order[k:]:                 # ranks that have not run in this step, R included
                f[j] = epoch
                f[W + j] = epoch
            awaited = host(f[:2 * W])
            assert (awaited >= epoch).all(), (f"rank {R} of {W} would wait at epoch {epoch}: round A {awaited[:W]}, "
                                              f"round B {awaited[W:]}")
            N.check(N.lib().b200_dp_adam_step(C.byref(self.comm[R]), N.ptr(self.m[R]), N.ptr(self.v[R]), self.n_params,
                                              self.n_total, LR, B1, B2, EPS, N.ptr(self.step[R]), N.ptr(self.epoch[R]),
                                              N.current_stream()), "b200_dp_adam_step")
            torch.cuda.synchronize()

    def assembled(self, moments):
        return torch.cat([moments[R][self.owned[R]] for R in range(self.W)])

    def state(self):
        return self.partials + self.params + self.m + self.v + self.step + self.epoch


def _dp_trajectory(W, n_params, n_total, order, worst, steps=3):
    """`steps` exchange steps of W emulated ranks, each checked against b200_adam_step on the rank-order sum (bit for
    bit) and against float64.  Returns the final state of every rank."""
    rng = np.random.default_rng([W, n_params])
    p0 = rng.standard_normal(n_params).astype(np.float32)
    m0 = (rng.standard_normal(n_params) * 1e-3).astype(np.float32)
    v0 = ((rng.standard_normal(n_params) * 1e-3) ** 2).astype(np.float32)
    ranks = Ranks(W, n_params, n_total, p0, m0, v0)
    ref = [torch.from_numpy(x).to(DEV) for x in (p0, m0, v0)]
    ref_step = torch.zeros(1, dtype=torch.int64, device=DEV)
    for s in range(1, steps + 1):
        parts = []
        for _ in range(W):
            q = (rng.standard_normal(n_total) * 10.0 ** rng.uniform(-4.0, 0.0, n_total)).astype(np.float32)
            q[rng.random(n_total) < 1.0 / 16] = 0.0
            parts.append(q)
        gsum = parts[0].copy()
        for q in parts[1:]:
            gsum = gsum + q                                    # ((p0 + p1) + p2) + ... in fp32, exactly
        gsum_d = torch.from_numpy(gsum).to(DEV)
        parts_d = [torch.from_numpy(q).to(DEV) for q in parts]
        for j in range(W):
            ranks.partials[j].copy_(parts_d[j])
        before = [host(t) for t in ref]
        ranks.run_step(order, s)
        _adam(ref[0], gsum_d, ref[1], ref[2], n_params, ref_step)
        torch.cuda.synchronize()
        where = f"W={W} n_params={n_params} order={'forward' if order[0] == 0 else 'reverse'} step {s}"
        for j in range(W):
            assert same(ranks.params[j], ref[0]), (where, "params of rank", j)
            assert same(ranks.partials[j][:n_params], parts_d[j][:n_params]), (where, "gradients of rank", j)
            assert same(ranks.partials[j][n_params:], gsum_d[n_params:]), (where, "loss tail of rank", j)
            o = ranks.owned[j]
            for name, mine, full in (("m", ranks.m[j], ref[1]), ("v", ranks.v[j], ref[2])):
                assert same(mine[o], full[o]), (where, name, "of rank", j, "on its slice", o)
                assert all_sentinel(mine[:o.start]) and all_sentinel(mine[o.stop:]), (where, name, "outside", o, j)
            assert int(ranks.step[j]) == s and int(ranks.epoch[j]) == s, (where, "step / epoch of rank", j)
        worst.step(host(ranks.params[0]), host(ranks.assembled(ranks.m)), host(ranks.assembled(ranks.v)),
                   adam_f64(*before, gsum[:n_params], s))
    return ranks.state()


@pytest.mark.gpu
@pytest.mark.parametrize("size", DP_SIZES)
@pytest.mark.parametrize("W", DP_WORLDS)
def test_dp_adam_emulated_ranks(W, size):
    """Three steps with fresh random partials, the ranks in forward and in reverse order: each rank's slice holds the
    rank-order fp32 sum, every rank's parameters equal b200_adam_step on that sum, the moments are written exactly on
    the rank's slice of the parameters, every partial buffer keeps its gradients and receives the summed loss tail,
    every step and epoch advance by one, and both orders give the same bytes.  A rank that wrote outside its slice
    would change what a later owner reads, so it fails in one of the two orders."""
    n_params, n_total = _dp_size(size)
    worst = Worst(f"dp W={W} {size} n_params={n_params} n_total={n_total}")
    fwd = _dp_trajectory(W, n_params, n_total, list(range(W)), worst)
    rev = _dp_trajectory(W, n_params, n_total, list(range(W))[::-1], worst)
    assert all(torch.equal(a, b) if a.dtype == torch.int64 else same(a, b) for a, b in zip(fwd, rev))
    worst.report()
