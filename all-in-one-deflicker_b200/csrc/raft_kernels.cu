// RAFT correlation: all-pairs volume + 4-level pyramid, and the 9x9 x 4-level bilinear lookup.
// Restates src/models/stage_1/core/corr.py:16-64 and core/utils/utils.py:57-71 (bilinear_sampler ->
// F.grid_sample(align_corners=True, zeros padding)) of the reference.
#include "common.cuh"

namespace b200 {

int simt_gemm_nn_scaled(const float* A_dim_major, const float* B_dim_major, float* C, int M, int N, int K, float scale,
                        cudaStream_t st);   // mlp_simt.cu: C[i][j] = scale * sum_d A[d][i] * B[d][j]

// F.avg_pool2d(x, 2, stride=2) on the last two dims of [planes][H][W] (floor mode)
__global__ void avgpool2_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t planes, int H, int W) {
  const int OH = H / 2, OW = W / 2;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= planes * OH * OW) return;
  const int ox = (int)(i % OW), oy = (int)((i / OW) % OH);
  const int64_t pl = i / ((int64_t)OW * OH);
  const float* s = x + (pl * H + 2 * oy) * W + 2 * ox;
  y[i] = (s[0] + s[1] + s[W] + s[W + 1]) * 0.25f;
}

// launcher for other translation units (conv_tma.cu pools feature maps with it)
int launch_avgpool2(const float* x, float* y, int64_t planes, int H, int W, cudaStream_t st) {
  const int64_t total = planes * (H / 2) * (W / 2);
  if (total <= 0) return B200_OK;
  avgpool2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, y, planes, H, W);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

struct LookupArgs {
  const float* level[4]; int LH[4], LW[4];   // sample 0's levels; sample b's lie sample_floats further on
  int64_t sample_floats;    // b200_corr_pyramid_floats(H1, W1)
  const float* coords;      // [B][2][H1][W1]  (x, y)
  float* out;               // [B][4*81][H1][W1]
  int B, H1, W1, radius;
};

// one thread per (pixel, level, tap).  Tap (i, j) of the window samples the level at
//   x = cx / 2^l + d_i ,  y = cy / 2^l + d_j ,  d = linspace(-r, r)      (corr.py:41-47: meshgrid(dy, dx)
// is added to (x, y), so the FIRST window index moves x) and lands in channel l*81 + i*9 + j.
__global__ void corr_lookup_kernel(LookupArgs a) {
  const int win = 2 * a.radius + 1, taps = win * win;
  const int64_t plane = (int64_t)a.H1 * a.W1;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)a.B * plane * 4 * taps) return;
  // pixel fastest so that writes are coalesced per output channel
  const int64_t pix = e % plane;
  const int tap = (int)((e / plane) % taps);
  const int l = (int)((e / (plane * taps)) % 4);
  const int b = (int)(e / (plane * taps * 4));
  const int i = tap / win, j = tap % win;
  const float cx = a.coords[((int64_t)b * 2 + 0) * plane + pix];
  const float cy = a.coords[((int64_t)b * 2 + 1) * plane + pix];
  const float inv = 1.0f / (float)(1 << l);
  const float x = cx * inv + (float)(i - a.radius);     // coords / 2**i is an exact power-of-two scaling
  const float y = cy * inv + (float)(j - a.radius);
  const int W = a.LW[l], H = a.LH[l];
  // bilinear_sampler: xgrid = 2*x/(W-1) - 1, then grid_sample(align_corners=True): ((g + 1) / 2) * (W - 1)
  const float gx = 2.0f * x / (float)(W - 1) - 1.0f, gy = 2.0f * y / (float)(H - 1) - 1.0f;
  const float ix = ((gx + 1.0f) / 2.0f) * (float)(W - 1), iy = ((gy + 1.0f) / 2.0f) * (float)(H - 1);
  // a 1-pixel-wide level makes (W-1) == 0: the reference's coordinates are inf/NaN there and F.grid_sample
  // returns NaN for the whole level (frames smaller than 128 px are unusable in the reference as well)
  if (!isfinite(ix) || !isfinite(iy)) { a.out[((int64_t)b * 4 * taps + l * taps + tap) * plane + pix] = nanf(""); return; }
  const float fx0 = floorf(ix), fy0 = floorf(iy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const float tx = ix - fx0, ty = iy - fy0;
  const float* src = a.level[l] + (int64_t)b * a.sample_floats + pix * H * W;
  auto at = [&](int yy, int xx) -> float { return (xx >= 0 && xx < W && yy >= 0 && yy < H) ? __ldg(src + (int64_t)yy * W + xx) : 0.f; };
  // ATen grid_sampler_2d: nw*(1-tx)(1-ty) + ne*tx(1-ty) + sw*(1-tx)ty + se*tx*ty
  const float v = at(y0, x0) * ((1.f - tx) * (1.f - ty)) + at(y0, x0 + 1) * (tx * (1.f - ty)) +
                  at(y0 + 1, x0) * ((1.f - tx) * ty) + at(y0 + 1, x0 + 1) * (tx * ty);
  a.out[((int64_t)b * 4 * taps + l * taps + tap) * plane + pix] = v;
}

// Tiled variant used for the standard radius 4: one block = 32 consecutive pixels x one level.  The 10x10
// neighbourhood the 81 bilinear taps of a pixel touch is staged once in shared memory (12x12 with margin) instead
// of 324 scattered loads; per-tap arithmetic is unchanged (same expressions as corr_lookup_kernel), taps that
// fall outside the staged window (non-finite or absurd coordinates) read global memory as before.
constexpr int LKW = 12;
__global__ void __launch_bounds__(256) corr_lookup_tiled_kernel(LookupArgs a) {
  __shared__ float win[32][LKW * LKW + 1];
  __shared__ int s_ox[32], s_oy[32];
  const int l = blockIdx.y, b = blockIdx.z, r = a.radius, wn = 2 * r + 1, taps = wn * wn;
  const int64_t plane = (int64_t)a.H1 * a.W1, pix0 = (int64_t)blockIdx.x * 32;
  const int W = a.LW[l], H = a.LH[l];
  const float inv = 1.0f / (float)(1 << l);
  if (threadIdx.x < 32) {
    const int64_t pix = pix0 + threadIdx.x;
    float cx = 0.f, cy = 0.f;
    if (pix < plane) { cx = a.coords[((int64_t)b * 2 + 0) * plane + pix]; cy = a.coords[((int64_t)b * 2 + 1) * plane + pix]; }
    const float fx = fminf(fmaxf(floorf(cx * inv), -1.0e6f), 1.0e6f), fy = fminf(fmaxf(floorf(cy * inv), -1.0e6f), 1.0e6f);
    s_ox[threadIdx.x] = (fx == fx ? (int)fx : 0) - r - 1;
    s_oy[threadIdx.x] = (fy == fy ? (int)fy : 0) - r - 1;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 32 * LKW * LKW; e += 256) {
    const int p = e / (LKW * LKW), k = e % (LKW * LKW);
    const int yy = s_oy[p] + k / LKW, xx = s_ox[p] + k % LKW;
    const int64_t pix = pix0 + p;
    float v = 0.f;
    if (pix < plane && xx >= 0 && xx < W && yy >= 0 && yy < H)
      v = __ldg(a.level[l] + (int64_t)b * a.sample_floats + pix * H * W + (int64_t)yy * W + xx);
    win[p][k] = v;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 32 * taps; e += 256) {
    const int p = e & 31, tap = e >> 5;
    const int64_t pix = pix0 + p;
    if (pix >= plane) continue;
    const int i = tap / wn, j = tap % wn;
    const float cx = a.coords[((int64_t)b * 2 + 0) * plane + pix];
    const float cy = a.coords[((int64_t)b * 2 + 1) * plane + pix];
    const float x = cx * inv + (float)(i - r);
    const float y = cy * inv + (float)(j - r);
    const float gx = 2.0f * x / (float)(W - 1) - 1.0f, gy = 2.0f * y / (float)(H - 1) - 1.0f;
    const float ix = ((gx + 1.0f) / 2.0f) * (float)(W - 1), iy = ((gy + 1.0f) / 2.0f) * (float)(H - 1);
    float* dst = a.out + ((int64_t)b * 4 * taps + l * taps + tap) * plane + pix;
    if (!isfinite(ix) || !isfinite(iy)) { *dst = nanf(""); continue; }
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const float tx = ix - fx0, ty = iy - fy0;
    float nw, ne, sw, se;
    const float rx = fx0 - (float)s_ox[p], ry = fy0 - (float)s_oy[p];
    if (rx >= 0.f && rx <= (float)(LKW - 2) && ry >= 0.f && ry <= (float)(LKW - 2)) {
      const float* wp = &win[p][(int)ry * LKW + (int)rx];
      nw = wp[0]; ne = wp[1]; sw = wp[LKW]; se = wp[LKW + 1];
    } else if (fabsf(fx0) < 1.0e9f && fabsf(fy0) < 1.0e9f) {
      const int x0 = (int)fx0, y0 = (int)fy0;
      const float* src = a.level[l] + (int64_t)b * a.sample_floats + pix * H * W;
      auto at = [&](int yy, int xx) -> float { return (xx >= 0 && xx < W && yy >= 0 && yy < H) ? __ldg(src + (int64_t)yy * W + xx) : 0.f; };
      nw = at(y0, x0); ne = at(y0, x0 + 1); sw = at(y0 + 1, x0); se = at(y0 + 1, x0 + 1);
    } else {
      nw = ne = sw = se = 0.f;
    }
    *dst = nw * ((1.f - tx) * (1.f - ty)) + ne * (tx * (1.f - ty)) + sw * ((1.f - tx) * ty) + se * (tx * ty);
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_corr_pyramid_floats(int32_t H8, int32_t W8) {
  int64_t total = 0, h = H8, w = W8;
  for (int l = 0; l < 4; ++l) { total += (int64_t)H8 * W8 * h * w; h /= 2; w /= 2; }
  return total;
}


int b200_corr_build(const float* fmap1, const float* fmap2, int32_t dim, int32_t H8, int32_t W8, float* pyramid, void* stream) {
  return b200_corr_build_batch(fmap1, fmap2, 1, dim, H8, W8, pyramid, stream);
}

int b200_corr_build_batch(const float* fmap1, const float* fmap2, int32_t batch, int32_t dim, int32_t H8, int32_t W8,
                          float* pyramid, void* stream) {
  B200_REQUIRE(fmap1 && fmap2 && pyramid && batch >= 1 && dim > 0 && H8 >= 8 && W8 >= 8, "bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int HW = H8 * W8;
  const int64_t fmap_floats = (int64_t)dim * HW, pyr_floats = b200_corr_pyramid_floats(H8, W8);
  for (int b = 0; b < batch; ++b) {
    // level 0: corr[p1][p2] = <f1[:, p1], f2[:, p2]> / sqrt(dim)        (corr.py:56-64)
    B200_PROPAGATE(simt_gemm_nn_scaled(fmap1 + b * fmap_floats, fmap2 + b * fmap_floats, pyramid + b * pyr_floats, HW, HW,
                                       dim, 1.0f / sqrtf((float)dim), st));
  }
  return b200_corr_pool_levels_batch(pyramid, batch, H8, W8, stream);
}

/* levels 1..3 of the pyramid from level 0: 2x2 average pooling over the target image (corr.py:22-25) */
int b200_corr_pool_levels(float* pyramid, int32_t H8, int32_t W8, void* stream) {
  return b200_corr_pool_levels_batch(pyramid, 1, H8, W8, stream);
}

int b200_corr_pool_levels_batch(float* pyramid, int32_t batch, int32_t H8, int32_t W8, void* stream) {
  B200_REQUIRE(pyramid && batch >= 1 && H8 >= 8 && W8 >= 8, "bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int HW = H8 * W8;
  const int64_t pyr_floats = b200_corr_pyramid_floats(H8, W8);
  for (int b = 0; b < batch; ++b) {
    float* cur = pyramid + b * pyr_floats;
    int h = H8, w = W8;
    for (int l = 1; l < 4; ++l) {
      float* nxt = cur + (int64_t)HW * h * w;
      const int64_t total = (int64_t)HW * (h / 2) * (w / 2);
      avgpool2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(cur, nxt, HW, h, w);
      B200_CHECK_LAUNCH();
      cur = nxt; h /= 2; w /= 2;
    }
  }
  return B200_OK;
}

int b200_corr_lookup(const float* pyramid, const float* coords, float* out, int32_t batch, int32_t H8, int32_t W8,
                     int32_t radius, void* stream) {
  B200_REQUIRE(batch == 1, "bad arguments (batch must be 1)");
  return b200_corr_lookup_batch(pyramid, coords, out, batch, H8, W8, radius, stream);
}

int b200_corr_lookup_batch(const float* pyramid, const float* coords, float* out, int32_t batch, int32_t H8, int32_t W8,
                           int32_t radius, void* stream) {
  B200_REQUIRE(pyramid && coords && out && batch >= 1 && batch <= 65535 && radius >= 1 && radius <= 8,
               "bad arguments (batch 1..65535, radius 1..8)");
  LookupArgs a{};
  const float* cur = pyramid;
  int h = H8, w = W8;
  for (int l = 0; l < 4; ++l) {
    a.level[l] = cur; a.LH[l] = h; a.LW[l] = w;
    cur += (int64_t)H8 * W8 * h * w; h /= 2; w /= 2;
  }
  a.sample_floats = b200_corr_pyramid_floats(H8, W8);
  a.coords = coords; a.out = out; a.B = batch; a.H1 = H8; a.W1 = W8; a.radius = radius;
  const int win = 2 * radius + 1;
  const int64_t total = (int64_t)batch * H8 * W8 * 4 * win * win;
  if (radius <= 4) {
    corr_lookup_tiled_kernel<<<dim3((unsigned)(((int64_t)H8 * W8 + 31) / 32), 4, batch), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  } else {
    corr_lookup_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  }
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
