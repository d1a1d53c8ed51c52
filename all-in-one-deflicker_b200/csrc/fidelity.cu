// Fidelity of frames to a reference (DESIGN §4f): for a frame O and a reference frame R, the SSIM sum over O's interior
// pixels and channels (Gaussian window, sigma 1.5, radius 5; the setting of skimage's structural_similarity with
// gaussian_weights=True, use_sample_covariance=False, data_range=1) and the squared-error sum over all of O's values.
// R of another size is resized to O's with cv2.resize(INTER_LINEAR) arithmetic in fp32 (resize_linear.cuh).
//
//   fidelity_kernel        one CTA per 16 x 32 output tile, the pairs' tiles back to back in one flat grid: the tile
//                          and its 5-pixel halo of O and R in shared memory, one channel at a time; the horizontal 11-tap pass over the five moment maps O, R, O^2, R^2,
//                          O R into shared memory, then the vertical pass and SSIM of two pixels per thread; per-CTA
//                          float64 partials of both sums
//   fidelity_final_kernel  one CTA per pair sums its partials
//
// The arithmetic is float64 with single IEEE operations (no fma contraction) in one fixed order, which the numpy
// restatement tests/fidelity_oracle.py reproduces.  Products of two fp32 values are exact in float64, so the moment
// maps carry no rounding.  The reduction order of a pair depends on its H and W only (tile by tile, the fixed CTA
// tree of cta_sum.cuh, then one CTA over the partials; no atomics): the sums are bit-identical across calls, graph
// replays, batch compositions and ranks.
#include <algorithm>

#include "common.cuh"
#include "cta_sum.cuh"
#include "resize_linear.cuh"

namespace b200 {

constexpr int kFidThreads = 256;
constexpr int kFidTileY = 16, kFidTileX = 32;
constexpr int kFidRadius = 5;
constexpr int kFidTaps = 2 * kFidRadius + 1;
constexpr int kFidInY = kFidTileY + 2 * kFidRadius, kFidInX = kFidTileX + 2 * kFidRadius;
constexpr int kFidMaxSide = 32768;

// w_k = exp(-k^2 / 4.5) / sum_j exp(-j^2 / 4.5), k = -5..5, the sum taken in k order: scipy.ndimage's
// gaussian_filter(sigma=1.5, truncate=3.5) weights, bit for bit
__constant__ double kFidW[kFidTaps] = {
    0x1.0d956b52a1d70p-10, 0x1.f1fe01ae5a5b8p-8, 0x1.26eb175d83f67p-5, 0x1.bff0fe8e98418p-4,
    0x1.b43c3f52b19f2p-3,  0x1.106560aa892c0p-2, 0x1.b43c3f52b19f2p-3, 0x1.bff0fe8e98418p-4,
    0x1.26eb175d83f67p-5,  0x1.f1fe01ae5a5b8p-8, 0x1.0d956b52a1d70p-10};
constexpr double kFidC1 = 0x1.a36e2eb1c432dp-14;    // 0.01^2
constexpr double kFidC2 = 0x1.d7dbf487fcb92p-11;    // 0.03^2

struct FidPairDev {
  const void* o;
  const void* r;
  int H, W, Hr, Wr, obits, rbits;
  int tiles_x, tiles;
  int tile0;                // first CTA of this pair in the flat grid
  int64_t pix_off;          // first pixel of this pair in the map
  int64_t part_off;         // first double of this pair's partials: [tiles] SSIM sums, then [tiles] squared errors
};
struct FidBatch {
  FidPairDev p[B200_FIDELITY_MAX_FRAMES];
  int n;
};

// v / 255 or v / 65535 rounded to fp32
__device__ __forceinline__ float decode(const void* img, int bits, int64_t i) {
  return bits == 8 ? __fdiv_rn((float)static_cast<const uint8_t*>(img)[i], 255.0f)
                   : __fdiv_rn((float)static_cast<const uint16_t*>(img)[i], 65535.0f);
}

__global__ void __launch_bounds__(kFidThreads) fidelity_kernel(FidBatch batch, double* __restrict__ partials,
                                                               float* __restrict__ map) {
  // the grid is every pair's tiles back to back: no CTA is launched for a smaller pair's missing tiles
  int pi = 0;
  while (pi + 1 < batch.n && (int)blockIdx.x >= batch.p[pi + 1].tile0) ++pi;
  const FidPairDev& pr = batch.p[pi];
  const int tile = (int)blockIdx.x - pr.tile0;
  __shared__ float sh_o[kFidInY][kFidInX], sh_r[kFidInY][kFidInX];
  __shared__ double sh_h[5][kFidInY][kFidTileX];
  __shared__ double sh_s[kFidThreads / 32], sh_e[kFidThreads / 32];
  const int H = pr.H, W = pr.W;
  const int y0 = (tile / pr.tiles_x) * kFidTileY, x0 = (tile % pr.tiles_x) * kFidTileX;
  const int tx = threadIdx.x % kFidTileX, ty = threadIdx.x / kFidTileX;      // pixels (ty, tx) and (ty + 8, tx)
  double s[2] = {0.0, 0.0}, e[2] = {0.0, 0.0};
  for (int c = 0; c < 3; ++c) {
    // the tile and its halo; zero outside the frame (only non-interior outputs read those)
    for (int i = threadIdx.x; i < kFidInY * kFidInX; i += kFidThreads) {
      const int ly = i / kFidInX, lx = i % kFidInX;
      const int y = y0 + ly - kFidRadius, x = x0 + lx - kFidRadius;
      float vo = 0.f, vr = 0.f;
      if (y >= 0 && y < H && x >= 0 && x < W) {
        vo = decode(pr.o, pr.obits, 3 * ((int64_t)y * W + x) + c);
        const void* rimg = pr.r;
        const int rb = pr.rbits, Wr = pr.Wr;
        vr = resize_sample<float>([&](int row, int col) { return decode(rimg, rb, 3 * ((int64_t)row * Wr + col) + c); },
                                  pr.Hr, pr.Wr, H, W, y, x);
      }
      sh_o[ly][lx] = vo;
      sh_r[ly][lx] = vr;
    }
    __syncthreads();
    // horizontal pass: h_m(row, x) = sum_k w_k m(row, x + k), k = -5..5 in order, for the five moment maps
    for (int i = threadIdx.x; i < kFidInY * kFidTileX; i += kFidThreads) {
      const int ly = i / kFidTileX, lx = i % kFidTileX;
      double ho = 0.0, hr = 0.0, hoo = 0.0, hrr = 0.0, hor = 0.0;
#pragma unroll
      for (int k = 0; k < kFidTaps; ++k) {
        const double o = (double)sh_o[ly][lx + k], r = (double)sh_r[ly][lx + k], w = kFidW[k];
        ho = add(ho, mul(w, o));
        hr = add(hr, mul(w, r));
        hoo = add(hoo, mul(w, mul(o, o)));
        hrr = add(hrr, mul(w, mul(r, r)));
        hor = add(hor, mul(w, mul(o, r)));
      }
      sh_h[0][ly][lx] = ho;
      sh_h[1][ly][lx] = hr;
      sh_h[2][ly][lx] = hoo;
      sh_h[3][ly][lx] = hrr;
      sh_h[4][ly][lx] = hor;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int ly = ty + j * (kFidTileY / 2);
      const int y = y0 + ly, x = x0 + tx;
      if (y >= H || x >= W) continue;
      const float o = sh_o[ly + kFidRadius][tx + kFidRadius], r = sh_r[ly + kFidRadius][tx + kFidRadius];
      const double d = __dsub_rn((double)o, (double)r);
      e[j] = add(e[j], mul(d, d));
      float v = __int_as_float(0x7fc00000);                                   // NaN outside the interior
      if (y >= kFidRadius && y < H - kFidRadius && x >= kFidRadius && x < W - kFidRadius) {
        double g[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int k = 0; k < kFidTaps; ++k) {
          const double w = kFidW[k];
#pragma unroll
          for (int m = 0; m < 5; ++m) g[m] = add(g[m], mul(w, sh_h[m][ly + k][tx]));
        }
        const double mo = g[0], mr = g[1];
        const double vo = __dsub_rn(g[2], mul(mo, mo)), vr = __dsub_rn(g[3], mul(mr, mr));
        const double cov = __dsub_rn(g[4], mul(mo, mr));
        const double a1 = add(mul(mul(2.0, mo), mr), kFidC1), a2 = add(mul(2.0, cov), kFidC2);
        const double b1 = add(add(mul(mo, mo), mul(mr, mr)), kFidC1), b2 = add(add(vo, vr), kFidC2);
        const double ssim = __ddiv_rn(mul(a1, a2), mul(b1, b2));
        s[j] = add(s[j], ssim);
        v = __double2float_rn(ssim);
      }
      if (map) map[3 * (pr.pix_off + (int64_t)y * W + x) + c] = v;
    }
    __syncthreads();                                                         // before the next channel's loads
  }
  const double ts = cta_sum<kFidThreads>(add(s[0], s[1]), sh_s);
  const double te = cta_sum<kFidThreads>(add(e[0], e[1]), sh_e);
  if (threadIdx.x == 0) {
    partials[pr.part_off + tile] = ts;
    partials[pr.part_off + pr.tiles + tile] = te;
  }
}

__global__ void __launch_bounds__(kFidThreads) fidelity_final_kernel(FidBatch batch, const double* __restrict__ partials,
                                                                     double* __restrict__ sums) {
  const FidPairDev& pr = batch.p[blockIdx.x];
  __shared__ double sh_s[kFidThreads / 32], sh_e[kFidThreads / 32];
  double s = 0.0, e = 0.0;
  for (int i = threadIdx.x; i < pr.tiles; i += kFidThreads) {
    s += partials[pr.part_off + i];
    e += partials[pr.part_off + pr.tiles + i];
  }
  s = cta_sum<kFidThreads>(s, sh_s);
  e = cta_sum<kFidThreads>(e, sh_e);
  if (threadIdx.x == 0) {
    sums[2 * blockIdx.x] = s;
    sums[2 * blockIdx.x + 1] = e;
  }
}

// Checks the descriptors and lays out the partials from byte 0 of the workspace.  Returns the bytes needed, or -1
// with the message set.
static int64_t plan_fidelity(const B200FidelityFrame* frames, int n, FidBatch* batch) {
  batch->n = n;
  if (!frames) {
    set_error("null frame table");
    return -1;
  }
  if (n < 1 || n > B200_FIDELITY_MAX_FRAMES) {
    set_error("%d frames: one call scores 1 to %d", n, B200_FIDELITY_MAX_FRAMES);
    return -1;
  }
  int64_t off = 0, pix = 0;
  int tile0 = 0;
  for (int i = 0; i < n; ++i) {
    const B200FidelityFrame& q = frames[i];
    if (!q.frame || !q.ref) {
      set_error("frame %d: null pointer", i);
      return -1;
    }
    if (q.H < kFidTaps || q.W < kFidTaps || q.H > kFidMaxSide || q.W > kFidMaxSide) {
      set_error("frame %d: %d x %d: SSIM's 11 x 11 window needs each side in [%d, %d]", i, q.H, q.W, kFidTaps,
                kFidMaxSide);
      return -1;
    }
    if (q.Hr <= 0 || q.Wr <= 0 || q.Hr > kFidMaxSide || q.Wr > kFidMaxSide) {
      set_error("frame %d: reference %d x %d: each side must be in [1, %d]", i, q.Hr, q.Wr, kFidMaxSide);
      return -1;
    }
    if ((q.bits != 8 && q.bits != 16) || (q.ref_bits != 8 && q.ref_bits != 16)) {
      set_error("frame %d: pixels of %d and %d bits; frames are uint8 (8) or uint16 (16)", i, q.bits, q.ref_bits);
      return -1;
    }
    if ((q.bits == 16 && (reinterpret_cast<uintptr_t>(q.frame) & 1)) ||
        (q.ref_bits == 16 && (reinterpret_cast<uintptr_t>(q.ref) & 1))) {
      set_error("frame %d: 16-bit frames must be 2-byte aligned", i);
      return -1;
    }
    FidPairDev& d = batch->p[i];
    d.o = q.frame;
    d.r = q.ref;
    d.H = q.H;
    d.W = q.W;
    d.Hr = q.Hr;
    d.Wr = q.Wr;
    d.obits = q.bits;
    d.rbits = q.ref_bits;
    d.tiles_x = (q.W + kFidTileX - 1) / kFidTileX;
    d.tiles = d.tiles_x * ((q.H + kFidTileY - 1) / kFidTileY);
    d.tile0 = tile0;
    tile0 += d.tiles;
    d.pix_off = pix;
    pix += (int64_t)q.H * q.W;
    d.part_off = off / (int64_t)sizeof(double);
    off += 2 * (int64_t)d.tiles * (int64_t)sizeof(double);
  }
  return off;
}

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_fidelity_workspace_bytes(const B200FidelityFrame* frames_host, int32_t n) {
  FidBatch batch;
  return plan_fidelity(frames_host, n, &batch);
}

int b200_fidelity(const B200FidelityFrame* frames_host, int32_t n, double* sums, float* ssim_map, void* ws,
                  int64_t ws_bytes, void* stream) {
  B200_REQUIRE(sums && ws, "null pointer (sums and the workspace are required; ssim_map may be NULL)");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 7) == 0, "workspace must be 8-byte aligned");
  FidBatch batch;
  const int64_t need = plan_fidelity(frames_host, n, &batch);
  if (need < 0) return B200_ERR_INVALID;
  if (ws_bytes < need) {
    set_error("workspace too small: need %lld bytes", (long long)need);
    return B200_ERR_WORKSPACE;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int grid = batch.p[n - 1].tile0 + batch.p[n - 1].tiles;
  double* partials = reinterpret_cast<double*>(ws);
  fidelity_kernel<<<grid, kFidThreads, 0, st>>>(batch, partials, ssim_map);
  B200_CHECK_LAUNCH();
  fidelity_final_kernel<<<n, kFidThreads, 0, st>>>(batch, partials, sums);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
