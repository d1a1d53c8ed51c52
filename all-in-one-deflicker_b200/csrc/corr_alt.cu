// RAFT correlation computed on the fly: the reference's AlternateCorrBlock (src/models/stage_1/core/corr.py:67-91,
// whose alt_cuda_corr extension is not shipped) with the output of CorrBlock.__call__, without the all-pairs volume.
//
// State (b200_corr_alt_floats): fmap1 and the four levels of fmap2, pixel-major ([pixels][dim]), so that one window
// position is one contiguous vector.  Level l of fmap2 is 2x2 floor-mode average pooling of level l-1, with the
// arithmetic of avgpool2_kernel; since pooling is linear, <fmap1[:, p], avgpool^l(fmap2)[:, q]> / sqrt(dim) is the
// value CorrBlock's pooled volume holds at (p, q).
//
// The lookup forms the dot products at the integer window positions, then the bilinear taps with the expressions of
// corr_lookup_tiled_kernel (raft_kernels.cu): same coordinate round trip, zero padding, NaN for non-finite coordinates
// and for levels 1 pixel wide or high.
#include <limits.h>

#include "common.cuh"

namespace b200 {

constexpr int ALT_TX = 16, ALT_TY = 4, ALT_TQ = ALT_TX * ALT_TY;   // query pixels of one CTA (a 16x4 tile)
constexpr int ALT_THREADS = 256;
constexpr int ALT_CC = 16;        // channels per staged chunk
constexpr int ALT_CS = 20;        // shared floats per staged chunk vector: 16 + 4 keeps neighbours' float4 reads conflict-free
constexpr int ALT_UMAX = 640;     // window positions of the largest staged union
constexpr int ALT_WMAX = 20;      // 2r + 4 for the largest radius, 8
constexpr int ALT_MAX_RADIUS = 8;

static int64_t alt_smem_bytes(int radius) {
  const int wm = 2 * radius + 4;
  return ((int64_t)ALT_TQ * wm * wm + ALT_TQ * ALT_CS + ALT_UMAX * ALT_CS) * 4;
}

// [dim][n] (channel-major encoder output) -> [n][dim]; sample blockIdx.z of x is x_stride floats on, of y y_stride
__global__ void alt_transpose_kernel(const float* __restrict__ x, float* __restrict__ y, int dim, int64_t n,
                                     int64_t x_stride, int64_t y_stride) {
  __shared__ float t[32][33];
  x += blockIdx.z * x_stride;
  y += blockIdx.z * y_stride;
  const int64_t p0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int c = c0 + k;
    const int64_t p = p0 + threadIdx.x;
    if (c < dim && p < n) t[k][threadIdx.x] = x[(int64_t)c * n + p];
  }
  __syncthreads();
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int64_t p = p0 + k;
    const int c = c0 + threadIdx.x;
    if (c < dim && p < n) y[p * dim + c] = t[threadIdx.x][k];
  }
}

// level l from level l-1, both pixel-major: F.avg_pool2d(2, stride=2) with avgpool2_kernel's (a + b + c + d) * 0.25;
// sample blockIdx.y is `stride` floats on in both
__global__ void alt_pool_kernel(const float* __restrict__ x, float* __restrict__ y, int dim, int H, int W, int64_t stride) {
  const int OH = H / 2, OW = W / 2;
  x += blockIdx.y * stride;
  y += blockIdx.y * stride;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)OH * OW * dim) return;
  const int c = (int)(i % dim);
  const int64_t q = i / dim;
  const int ox = (int)(q % OW), oy = (int)(q / OW);
  const float* s = x + ((int64_t)(2 * oy) * W + 2 * ox) * dim + c;
  const int64_t row = (int64_t)W * dim;
  y[i] = (s[0] + s[dim] + s[row] + s[row + dim]) * 0.25f;
}

struct AltArgs {
  const float* f1;               // [H1*W1][dim]  (sample 0; sample b's state is b * state_floats further on)
  const float* level[4];         // [LH*LW][dim]
  int LH[4], LW[4];
  int64_t state_floats;          // b200_corr_alt_floats(dim, H1, W1)
  const float* coords;           // [B][2][H1][W1]  (x, y)
  float* out;                    // [B][4*(2r+1)^2][H1][W1]
  int H1, W1, dim, radius;
  float scale;                   // 1 / sqrt(dim)
};

// corr_lookup_tiled_kernel's sampling coordinate of a window offset: x = c / 2^l + off, then the reference's fp32 round
// trip through grid_sample's normalised grid (align_corners=True)
__device__ __forceinline__ float alt_sample(float c, float inv, int off, int n) {
  const float x = c * inv + (float)off;
  const float g = 2.0f * x / (float)(n - 1) - 1.0f;
  return ((g + 1.0f) / 2.0f) * (float)(n - 1);
}

__device__ __forceinline__ float alt_chunk_dot(const float4 (&f)[4], const float4 (&b)[4]) {
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    acc = fmaf(f[k].x, b[k].x, acc); acc = fmaf(f[k].y, b[k].y, acc);
    acc = fmaf(f[k].z, b[k].z, acc); acc = fmaf(f[k].w, b[k].w, acc);
  }
  return acc;
}

// One dot product straight from global memory, summed in the same order as the staged path (16-channel chunks, each an
// fma chain), so that a value does not depend on whether its window was staged.
__device__ float alt_dot_global(const float* __restrict__ f1, const float* __restrict__ v, int dim) {
  float total = 0.f;
  for (int c0 = 0; c0 < dim; c0 += ALT_CC) {
    float4 f[4], b[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      f[k] = __ldg(reinterpret_cast<const float4*>(f1 + c0) + k);
      b[k] = __ldg(reinterpret_cast<const float4*>(v + c0) + k);
    }
    const float acc = alt_chunk_dot(f, b);
    total = c0 == 0 ? acc : total + acc;
  }
  return total;
}

// Dot products of one window row of one query pixel with one 16-channel chunk, added into the shared results
// (row stride ALT_TQ: the lanes of a warp are consecutive query pixels).
template <bool STAGED>
__device__ __forceinline__ void alt_row_chunk(const float4 (&f)[4], const float* src, int64_t stride, int nx, float* drow,
                                              bool first) {
#pragma unroll 4
  for (int a = 0; a < ALT_WMAX; ++a) {
    if (a >= nx) break;
    const float4* v = reinterpret_cast<const float4*>(src + a * stride);
    float4 b[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) b[k] = STAGED ? v[k] : __ldg(v + k);
    const float acc = alt_chunk_dot(f, b);
    drow[a * ALT_TQ] = first ? acc : drow[a * ALT_TQ] + acc;
  }
}

// One CTA = a 16x4 tile of query pixels at one level (blockIdx.y) of one sample (blockIdx.z).
//  1. each query pixel's window: the integer positions its taps' corners touch (floor of the first and the last tap's
//     coordinate, one more; at most 2r+4 per axis), clipped to the level;
//  2. the dot products at those positions, 16 channels at a time: fmap1 chunks of the tile, and the union of the
//     windows when it has at most ALT_UMAX positions, are staged in shared memory; otherwise (large or incoherent
//     flow) the positions are read from global memory;
//  3. the taps, from the shared dot products; a corner outside its pixel's window (only when the coordinate round trip
//     moves a tap by more than the window's margin) is computed from global memory.
__global__ void __launch_bounds__(ALT_THREADS) corr_alt_lookup_kernel(AltArgs a) {
  extern __shared__ float4 alt_smem[];
  const int r = a.radius, wn = 2 * r + 1, taps = wn * wn, wm = 2 * r + 4, dim = a.dim;
  float* sdot = reinterpret_cast<float*>(alt_smem);        // [wm][wm][ALT_TQ]
  float* sf1 = sdot + ALT_TQ * wm * wm;                    // [ALT_TQ][ALT_CS]
  float* su = sf1 + ALT_TQ * ALT_CS;                       // [ALT_UMAX][ALT_CS]
  __shared__ int s_wx[ALT_TQ], s_wy[ALT_TQ], s_nx[ALT_TQ], s_ny[ALT_TQ];
  __shared__ float s_cx[ALT_TQ], s_cy[ALT_TQ];
  __shared__ int s_u[4];
  const int l = blockIdx.y;
  const int tiles_x = (a.W1 + ALT_TX - 1) / ALT_TX;
  const int tx0 = (int)(blockIdx.x % tiles_x) * ALT_TX, ty0 = (int)(blockIdx.x / tiles_x) * ALT_TY;
  const int64_t plane = (int64_t)a.H1 * a.W1;
  const int W = a.LW[l], H = a.LH[l];
  const float inv = 1.0f / (float)(1 << l);
  const int64_t sample = (int64_t)blockIdx.z * a.state_floats;
  const float* f1 = a.f1 + sample;
  const float* lvl = a.level[l] + sample;
  const float* coords = a.coords + (int64_t)blockIdx.z * 2 * plane;
  float* out = a.out + (int64_t)blockIdx.z * 4 * taps * plane;
  if (threadIdx.x == 0) { s_u[0] = s_u[1] = INT_MAX; s_u[2] = s_u[3] = INT_MIN; }
  __syncthreads();
  if (threadIdx.x < ALT_TQ) {
    const int p = threadIdx.x, px = tx0 + p % ALT_TX, py = ty0 + p / ALT_TX;
    int wx = 0, wy = 0, nx = 0, ny = 0;
    float cx = 0.f, cy = 0.f;
    if (px < a.W1 && py < a.H1) {
      const int64_t pix = (int64_t)py * a.W1 + px;
      cx = coords[pix]; cy = coords[plane + pix];
      const float x0 = alt_sample(cx, inv, -r, W), x1 = alt_sample(cx, inv, r, W);
      const float y0 = alt_sample(cy, inv, -r, H), y1 = alt_sample(cy, inv, r, H);
      if (isfinite(x0) && isfinite(x1) && isfinite(y0) && isfinite(y1)) {
        const float xl = fmaxf(floorf(x0), 0.f), xh = fminf(floorf(x1) + 1.f, (float)(W - 1));
        const float yl = fmaxf(floorf(y0), 0.f), yh = fminf(floorf(y1) + 1.f, (float)(H - 1));
        if (xl <= xh && yl <= yh) {
          wx = (int)xl; wy = (int)yl;
          nx = min((int)xh - wx + 1, wm); ny = min((int)yh - wy + 1, wm);
          atomicMin(&s_u[0], wx); atomicMin(&s_u[1], wy);
          atomicMax(&s_u[2], wx + nx - 1); atomicMax(&s_u[3], wy + ny - 1);
        }
      }
    }
    s_wx[p] = wx; s_wy[p] = wy; s_nx[p] = nx; s_ny[p] = ny; s_cx[p] = cx; s_cy[p] = cy;
  }
  __syncthreads();
  const int ux0 = s_u[0], uy0 = s_u[1];
  if (s_u[2] >= ux0) {                                     // some window lies (partly) inside the level
    const int uw = s_u[2] - ux0 + 1, uh = s_u[3] - uy0 + 1;
    const bool staged = (int64_t)uw * uh <= ALT_UMAX;
    for (int c0 = 0; c0 < dim; c0 += ALT_CC) {
      if (c0) __syncthreads();                             // the previous chunk is consumed
      {
        static_assert(ALT_TQ * 4 == ALT_THREADS, "one float4 of the fmap1 chunk per thread");
        const int p = threadIdx.x >> 2, k = threadIdx.x & 3, px = tx0 + p % ALT_TX, py = ty0 + p / ALT_TX;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (px < a.W1 && py < a.H1) v = __ldg(reinterpret_cast<const float4*>(f1 + ((int64_t)py * a.W1 + px) * dim + c0) + k);
        reinterpret_cast<float4*>(sf1 + p * ALT_CS)[k] = v;
      }
      if (staged) {
        for (int e = threadIdx.x; e < uw * uh * 4; e += ALT_THREADS) {
          const int pos = e >> 2, k = e & 3;
          const int yy = uy0 + pos / uw, xx = ux0 + pos % uw;
          reinterpret_cast<float4*>(su + pos * ALT_CS)[k] =
              __ldg(reinterpret_cast<const float4*>(lvl + ((int64_t)yy * W + xx) * dim + c0) + k);
        }
      }
      __syncthreads();
      for (int e = threadIdx.x; e < ALT_TQ * wm; e += ALT_THREADS) {
        const int p = e % ALT_TQ, b = e / ALT_TQ;
        if (b >= s_ny[p]) continue;
        const int yy = s_wy[p] + b, xx = s_wx[p];
        float4 f[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) f[k] = reinterpret_cast<const float4*>(sf1 + p * ALT_CS)[k];
        float* drow = sdot + (b * wm) * ALT_TQ + p;
        if (staged)
          alt_row_chunk<true>(f, su + ((yy - uy0) * uw + (xx - ux0)) * ALT_CS, ALT_CS, s_nx[p], drow, c0 == 0);
        else
          alt_row_chunk<false>(f, lvl + ((int64_t)yy * W + xx) * dim + c0, dim, s_nx[p], drow, c0 == 0);
      }
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < ALT_TQ * taps; e += ALT_THREADS) {
    const int p = e % ALT_TQ, tap = e / ALT_TQ, px = tx0 + p % ALT_TX, py = ty0 + p / ALT_TX;
    if (px >= a.W1 || py >= a.H1) continue;
    const int64_t pix = (int64_t)py * a.W1 + px;
    const int i = tap / wn, j = tap % wn;
    const float ix = alt_sample(s_cx[p], inv, i - r, W), iy = alt_sample(s_cy[p], inv, j - r, H);
    float* dst = out + (int64_t)(l * taps + tap) * plane + pix;
    if (!isfinite(ix) || !isfinite(iy)) { *dst = nanf(""); continue; }
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const float tx = ix - fx0, ty = iy - fy0;
    const int wx = s_wx[p], wy = s_wy[p], nx = s_nx[p], ny = s_ny[p];
    auto at = [&](float yf, float xf) -> float {
      if (!(xf >= 0.f && xf <= (float)(W - 1) && yf >= 0.f && yf <= (float)(H - 1))) return 0.f;   // zero padding
      const int xi = (int)xf, yi = (int)yf, dx = xi - wx, dy = yi - wy;
      if (dx >= 0 && dx < nx && dy >= 0 && dy < ny) return sdot[(dy * wm + dx) * ALT_TQ + p] * a.scale;
      return alt_dot_global(f1 + pix * a.dim, lvl + ((int64_t)yi * W + xi) * a.dim, a.dim) * a.scale;
    };
    const float nw = at(fy0, fx0), ne = at(fy0, fx0 + 1.f), sw = at(fy0 + 1.f, fx0), se = at(fy0 + 1.f, fx0 + 1.f);
    *dst = nw * ((1.f - tx) * (1.f - ty)) + ne * (tx * (1.f - ty)) + sw * ((1.f - tx) * ty) + se * (tx * ty);
  }
}

// floats of fmap1 and of the four fmap2 levels, each pixel-major; -1 for a geometry the kernels do not take
static int64_t alt_layout(int dim, int H8, int W8, int64_t off[5]) {
  if (dim <= 0 || dim % ALT_CC != 0 || H8 < 8 || W8 < 8) return -1;
  int64_t n = (int64_t)H8 * W8 * dim;
  off[0] = 0;
  int h = H8, w = W8;
  for (int l = 0; l < 4; ++l) {
    off[l + 1] = n;
    n += (int64_t)h * w * dim;
    h /= 2; w /= 2;
  }
  return n;
}

static int ensure_alt_attrs() {
  static bool done_dev[64] = {};
  int dev = 0;
  B200_CHECK_CUDA(cudaGetDevice(&dev));
  B200_REQUIRE(dev >= 0 && dev < 64, "device ordinal %d out of range", dev);
  if (done_dev[dev]) return B200_OK;
  B200_CHECK_CUDA(cudaFuncSetAttribute(corr_alt_lookup_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)alt_smem_bytes(ALT_MAX_RADIUS)));
  done_dev[dev] = true;
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_corr_alt_floats(int32_t dim, int32_t H8, int32_t W8) {
  int64_t off[5];
  return alt_layout(dim, H8, W8, off);
}

int b200_corr_alt_build(const float* fmap1, const float* fmap2, int32_t dim, int32_t H8, int32_t W8, float* state,
                        void* stream) {
  return b200_corr_alt_build_batch(fmap1, fmap2, 1, dim, H8, W8, state, stream);
}

int b200_corr_alt_build_batch(const float* fmap1, const float* fmap2, int32_t batch, int32_t dim, int32_t H8, int32_t W8,
                              float* state, void* stream) {
  int64_t off[5];
  B200_REQUIRE(fmap1 && fmap2 && state, "b200_corr_alt_build: null pointer");
  B200_REQUIRE(batch >= 1 && batch <= 65535, "b200_corr_alt_build: batch must be 1..65535 (got %d)", batch);
  const int64_t floats = alt_layout(dim, H8, W8, off);
  B200_REQUIRE(floats > 0, "b200_corr_alt_build: dim must be a positive multiple of %d and H8, W8 >= 8 "
               "(got dim %d, %dx%d)", ALT_CC, dim, H8, W8);
  B200_REQUIRE(reinterpret_cast<uintptr_t>(state) % 16 == 0, "b200_corr_alt_build: state must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t n = (int64_t)H8 * W8;
  const dim3 grid((unsigned)((n + 31) / 32), (unsigned)((dim + 31) / 32), (unsigned)batch);
  alt_transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(fmap1, state + off[0], dim, n, dim * n, floats);
  B200_CHECK_LAUNCH();
  alt_transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(fmap2, state + off[1], dim, n, dim * n, floats);
  B200_CHECK_LAUNCH();
  int h = H8, w = W8;
  for (int l = 1; l < 4; ++l) {
    const int64_t total = (int64_t)(h / 2) * (w / 2) * dim;
    alt_pool_kernel<<<dim3((unsigned)((total + 255) / 256), (unsigned)batch), 256, 0, st>>>(state + off[l], state + off[l + 1],
                                                                                          dim, h, w, floats);
    B200_CHECK_LAUNCH();
    h /= 2; w /= 2;
  }
  return B200_OK;
}

int b200_corr_alt_lookup(const float* state, const float* coords, float* out, int32_t dim, int32_t batch, int32_t H8,
                         int32_t W8, int32_t radius, void* stream) {
  B200_REQUIRE(batch == 1, "b200_corr_alt_lookup: batch must be 1 (got %d)", batch);
  return b200_corr_alt_lookup_batch(state, coords, out, dim, batch, H8, W8, radius, stream);
}

int b200_corr_alt_lookup_batch(const float* state, const float* coords, float* out, int32_t dim, int32_t batch, int32_t H8,
                               int32_t W8, int32_t radius, void* stream) {
  int64_t off[5];
  B200_REQUIRE(state && coords && out, "b200_corr_alt_lookup: null pointer");
  B200_REQUIRE(batch >= 1 && batch <= 65535, "b200_corr_alt_lookup: batch must be 1..65535 (got %d)", batch);
  B200_REQUIRE(radius >= 1 && radius <= ALT_MAX_RADIUS, "b200_corr_alt_lookup: radius must be 1..%d (got %d)",
               ALT_MAX_RADIUS, radius);
  const int64_t floats = alt_layout(dim, H8, W8, off);
  B200_REQUIRE(floats > 0, "b200_corr_alt_lookup: dim must be a positive multiple of %d and "
               "H8, W8 >= 8 (got dim %d, %dx%d)", ALT_CC, dim, H8, W8);
  B200_REQUIRE(reinterpret_cast<uintptr_t>(state) % 16 == 0, "b200_corr_alt_lookup: state must be 16-byte aligned");
  B200_PROPAGATE(ensure_alt_attrs());
  AltArgs a{};
  a.f1 = state + off[0];
  int h = H8, w = W8;
  for (int l = 0; l < 4; ++l) {
    a.level[l] = state + off[l + 1]; a.LH[l] = h; a.LW[l] = w;
    h /= 2; w /= 2;
  }
  a.state_floats = floats;
  a.coords = coords; a.out = out; a.H1 = H8; a.W1 = W8; a.dim = dim; a.radius = radius;
  a.scale = 1.0f / sqrtf((float)dim);
  const unsigned tiles = (unsigned)(((W8 + ALT_TX - 1) / ALT_TX) * ((H8 + ALT_TY - 1) / ALT_TY));
  corr_alt_lookup_kernel<<<dim3(tiles, 4, (unsigned)batch), ALT_THREADS, (size_t)alt_smem_bytes(radius),
                           reinterpret_cast<cudaStream_t>(stream)>>>(a);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
