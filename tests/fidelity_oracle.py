"""Float64 numpy restatement of the fidelity metric (DESIGN §4f) that csrc/fidelity.cu computes: SSIM with the
Gaussian window of skimage's structural_similarity(gaussian_weights=True, sigma=1.5, use_sample_covariance=False,
data_range=1) and the squared error, in the kernel's operation order, and the kernel's fixed-order reduction.  The
reference resize is oracle/stage2_io_oracle's resize_linear_f32 (pinned against cv2.resize) on the decoded fp32 values.
`ssim_plain` is a second, independent form on scipy.ndimage.gaussian_filter that stands in for skimage.

TEST INFRASTRUCTURE ONLY: nothing in the product imports this module."""
import math

import numpy as np

from oracle import stage2_io_oracle as SO
import flicker_oracle as FO

RADIUS = 5
TILE_Y, TILE_X = 16, 32
C1, C2 = 0.01 ** 2, 0.03 ** 2


def taps():
    """w_k = exp(-k^2 / 4.5) / sum_j exp(-j^2 / 4.5), k = -5..5, the sum in k order."""
    e = [math.exp(-k * k / 4.5) for k in range(-RADIUS, RADIUS + 1)]
    s = 0.0
    for v in e:
        s += v
    return np.array([v / s for v in e])


def decode(img):
    """uint8 / uint16 (H, W, 3) -> v / 255 or v / 65535 rounded to fp32."""
    return FO.decode(img).astype(np.float32)


def reference_at(ref, H, W):
    """R decoded to fp32 and resized to (H, W) with cv2's INTER_LINEAR arithmetic (as is at its own size)."""
    r = decode(ref)
    if r.shape[:2] == (H, W):
        return r
    return SO.resize_linear_f32(r, W, H).reshape(H, W, 3)


def ssim_map(frame, ref):
    """(H, W, 3) float64 SSIM in the kernel's order, NaN outside the interior."""
    o = decode(frame).astype(np.float64)
    H, W = o.shape[:2]
    if H < 2 * RADIUS + 1 or W < 2 * RADIUS + 1:
        raise ValueError("%d x %d: SSIM's 11 x 11 window needs each side >= 11" % (H, W))
    r = reference_at(ref, H, W).astype(np.float64)
    w = taps()
    out = np.full((H, W, 3), np.nan)
    for c in range(3):
        maps = [o[..., c], r[..., c], o[..., c] * o[..., c], r[..., c] * r[..., c], o[..., c] * r[..., c]]
        g = []
        for m in maps:
            p = np.zeros((H + 2 * RADIUS, W + 2 * RADIUS))
            p[RADIUS:-RADIUS, RADIUS:-RADIUS] = m
            h = np.zeros((H + 2 * RADIUS, W))
            for k in range(2 * RADIUS + 1):
                h = h + w[k] * p[:, k:k + W]
            v = np.zeros((H, W))
            for k in range(2 * RADIUS + 1):
                v = v + w[k] * h[k:k + H]
            g.append(v)
        mo, mr = g[0], g[1]
        vo, vr, cov = g[2] - mo * mo, g[3] - mr * mr, g[4] - mo * mr
        a1, a2 = (2.0 * mo) * mr + C1, 2.0 * cov + C2
        b1, b2 = (mo * mo + mr * mr) + C1, (vo + vr) + C2
        s = (a1 * a2) / (b1 * b2)
        out[RADIUS:H - RADIUS, RADIUS:W - RADIUS, c] = s[RADIUS:H - RADIUS, RADIUS:W - RADIUS]
    return out


def error_map(frame, ref):
    """(H, W) float64: per pixel ((0 + d_0^2) + d_1^2) + d_2^2, d = O - R."""
    o = decode(frame).astype(np.float64)
    r = reference_at(ref, *o.shape[:2]).astype(np.float64)
    d = o - r
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _tile_sum(values):
    """fidelity.cu's float64 sum of an (H, W) map: per 16 x 32 tile, thread (ty, tx) adds rows ty and ty + 8, the CTA
    tree of cta_sum.cuh, then one CTA over the tile partials in tile order."""
    H, W = values.shape
    ty, tx = -(-H // TILE_Y), -(-W // TILE_X)
    p = np.zeros((ty * TILE_Y, tx * TILE_X))
    p[:H, :W] = values
    t = p.reshape(ty, TILE_Y, tx, TILE_X).transpose(0, 2, 1, 3).reshape(ty * tx, TILE_Y, TILE_X)
    acc = (t[:, :TILE_Y // 2] + t[:, TILE_Y // 2:]).reshape(ty * tx, FO.THREADS)
    parts = FO._cta_sum(acc)
    padded = np.zeros(-(-parts.size // FO.THREADS) * FO.THREADS)
    padded[:parts.size] = parts
    acc = np.zeros(FO.THREADS)
    for row in padded.reshape(-1, FO.THREADS):
        acc = acc + row
    return float(FO._cta_sum(acc))


def frame_sums(frame, ref, smap=None):
    """(SSIM sum over the interior and channels, squared-error sum over the frame) in the kernel's order."""
    s = ssim_map(frame, ref) if smap is None else smap
    per_pixel = np.nan_to_num((s[..., 0] + s[..., 1]) + s[..., 2], nan=0.0)
    return _tile_sum(per_pixel), _tile_sum(error_map(frame, ref))


def frame_values(frame, ref):
    """(S(t), PSNR(t)) of one frame, PSNR None when the frame equals the reference."""
    H, W = frame.shape[:2]
    ssum, sse = frame_sums(frame, ref)
    return ssum / (3.0 * (H - 2 * RADIUS) * (W - 2 * RADIUS)), (
        None if sse == 0 else 10.0 * math.log10(1.0 / (sse / (3.0 * H * W))))


def ssim_plain(frame, ref):
    """Mean SSIM the way skimage computes it (gaussian_filter(sigma=1.5, truncate=3.5) on each moment, 5-pixel
    crop), in numpy's own order: a second form to hold the restatement to."""
    from scipy.ndimage import gaussian_filter
    o = decode(frame).astype(np.float64)
    r = reference_at(ref, *o.shape[:2]).astype(np.float64)
    f = lambda a: gaussian_filter(a, sigma=1.5, truncate=3.5)
    vals = []
    for c in range(3):
        x, y = o[..., c], r[..., c]
        ux, uy, uxx, uyy, uxy = f(x), f(y), f(x * x), f(y * y), f(x * y)
        vx, vy, vxy = uxx - ux * ux, uyy - uy * uy, uxy - ux * uy
        S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
        vals.append(S[RADIUS:-RADIUS, RADIUS:-RADIUS].mean())
    return float(np.mean(vals))


def texture(rng, H, W, bits=8):
    """A test frame: a smooth random texture plus noise, so that the local moments vary; (H, W, 3) uint8 or
    uint16."""
    import cv2
    top = 255 if bits == 8 else 65535
    base = rng.random((max(2, H // 8), max(2, W // 8), 3)).astype(np.float32)
    img = cv2.resize(base, (W, H), interpolation=cv2.INTER_LINEAR).reshape(H, W, 3)
    img = np.clip(img + 0.05 * rng.standard_normal((H, W, 3)), 0, 1)
    return np.round(img * top).astype(np.uint8 if bits == 8 else np.uint16)
