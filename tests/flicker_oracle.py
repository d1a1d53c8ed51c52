"""Float64 numpy restatement of the temporal warping error (DESIGN §4e) that csrc/warp_error.cu computes, in the
kernel's operation order, and of the kernel's fixed-order reduction.  The flow resize is oracle/stage2_io_oracle's
resize_linear_f32 (pinned against cv2.resize), followed by the geometric scaling: x by W / Wf, y by H / Hf, in fp32.

TEST INFRASTRUCTURE ONLY: nothing in the product imports this module."""
import numpy as np

from oracle import stage2_io_oracle as SO

THREADS, MAX_BLOCKS = 256, 1024


def decode(img):
    """uint8 / uint16 (H, W, 3) -> v / 255 or v / 65535 rounded to fp32, as float64."""
    den = np.float32(255 if img.dtype == np.uint8 else 65535)
    return (img.astype(np.float32) / den).astype(np.float64)


def resize_flow(flow, H, W):
    """A (Hf, Wf, 2) fp32 flow at (H, W): resized with cv2's INTER_LINEAR arithmetic, x scaled by W / Wf and y by
    H / Hf (fp32); returned as is at its own size."""
    flow = np.asarray(flow, np.float32)
    Hf, Wf = flow.shape[:2]
    if (Hf, Wf) == (H, W):
        return flow.copy()
    r = SO.resize_linear_f32(flow, W, H)
    return np.stack([r[..., 0] * np.float32(W / Wf), r[..., 1] * np.float32(H / Hf)], axis=-1).astype(np.float32)


def _lerp2(v00, v01, v10, v11, ax, bx, ay, by):
    return (v00 * bx + v01 * ax) * by + (v10 * bx + v11 * ax) * ay


def warp_maps(f0, f1, fwd, bwd, margins=False):
    """Per pixel of frame t: the float64 error sum_c (O_t - W^)^2 where q = p + F(p) lies in the frame (0 elsewhere)
    and the mask.  With margins=True also rhs - lhs of the occlusion test (NaN where q is outside)."""
    H, W = f0.shape[:2]
    F = resize_flow(fwd, H, W).astype(np.float64)
    B = resize_flow(bwd, H, W).astype(np.float64)
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    fx, fy = F[..., 0], F[..., 1]
    with np.errstate(invalid="ignore"):
        qx, qy = xx + fx, yy + fy
        inside = (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
    qx, qy = np.where(inside, qx, 0.0), np.where(inside, qy, 0.0)
    x0, y0 = np.floor(qx).astype(np.int64), np.floor(qy).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    ax, ay = qx - x0, qy - y0
    bx, by = 1.0 - ax, 1.0 - ay
    taps = lambda img: (img[y0, x0], img[y0, x1], img[y1, x0], img[y1, x1])
    k = lambda a: a[..., None]
    with np.errstate(invalid="ignore", over="ignore"):
        Bt = _lerp2(*taps(B), k(ax), k(bx), k(ay), k(by))
        sx, sy = fx + Bt[..., 0], fy + Bt[..., 1]
        lhs = sx * sx + sy * sy
        rhs = 0.01 * ((fx * fx + fy * fy) + (Bt[..., 0] * Bt[..., 0] + Bt[..., 1] * Bt[..., 1])) + 0.5
        mask = inside & (lhs <= rhs)
    O0, O1 = decode(f0), decode(f1)
    d = O0 - _lerp2(*taps(O1), k(ax), k(bx), k(ay), k(by))
    err = np.where(inside, (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2], 0.0)
    if margins:
        return err, mask, np.where(inside, rhs - lhs, np.nan)
    return err, mask


def pair_sums(f0, f1, fwd, bwd):
    """(masked squared-error sum, |M|) of one pair, the error rounded to fp32 per pixel as the kernel sums it."""
    err, mask = warp_maps(f0, f1, fwd, bwd)
    return float(np.sum(err.astype(np.float32).astype(np.float64)[mask])), float(mask.sum())


def pair_value(f0, f1, fwd, bwd):
    sse, n = pair_sums(f0, f1, fwd, bwd)
    return sse / (3 * n) if n else float("nan")


def _cta_sum(v):
    """cta_sum.cuh over the last axis (256 threads): xor butterfly in each warp, then over the 8 warp sums."""
    lanes = np.arange(32)
    w = v.reshape(v.shape[:-1] + (THREADS // 32, 32))
    for o in (16, 8, 4, 2, 1):
        w = w + w[..., lanes ^ o]
    z = np.zeros(v.shape[:-1] + (32,))
    z[..., :THREADS // 32] = w[..., 0]
    for o in (16, 8, 4, 2, 1):
        z = z + z[..., lanes ^ o]
    return z[..., 0]


def blocks_of(pixels):
    return min(-(-pixels // THREADS), MAX_BLOCKS)


def kernel_order_sum(values):
    """float64 sum of per-pixel values in warp_error.cu's order: each thread's grid-stride sequence, the CTA tree per
    block, then one CTA over the block partials."""
    values = np.asarray(values, np.float64).reshape(-1)
    G = blocks_of(values.size)
    span = G * THREADS
    padded = np.zeros(-(-values.size // span) * span)
    padded[:values.size] = values
    acc = np.zeros((G, THREADS))
    for row in padded.reshape(-1, G, THREADS):
        acc = acc + row
    parts = _cta_sum(acc)
    padded = np.zeros(-(-G // THREADS) * THREADS)
    padded[:G] = parts
    acc = np.zeros(THREADS)
    for row in padded.reshape(-1, THREADS):
        acc = acc + row
    return float(_cta_sum(acc))
