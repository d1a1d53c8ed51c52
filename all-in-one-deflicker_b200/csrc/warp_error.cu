// Temporal warping error of frame pairs (DESIGN §4e): for frames t, t+1 of a sequence and the flow pre-pass's forward
// flow F (t -> t+1) and backward flow B (t+1 -> t), the squared difference between frame t and frame t+1 sampled at
// q = p + F(p), summed over the pixels p that pass the forward-backward occlusion test, and the number of those pixels.
//
//   warp_flow_resize_kernel  flows of another resolution: cv2.resize(INTER_LINEAR) in fp32 (resize_linear.cuh), then
//                            x times W / Wf and y times H / Hf (the geometric scaling, not resize_flow's swapped one)
//   warp_error_kernel        per pixel: q, bilinear samples of frame t+1 and of B at q, the mask, the error; per-CTA
//                            float64 partials of the masked error and of the mask count
//   warp_error_final_kernel  one CTA per pair sums its partials
//
// Per pixel the arithmetic is float64 with single IEEE operations (no fma contraction), so a numpy restatement in the
// same order reproduces the mask and the error; the error is rounded to fp32 once and that fp32 value is what the
// partials sum.  The reduction order of a pair depends on its H * W only (grid-stride, then the fixed CTA tree of
// cta_sum.cuh, then one CTA over the partials; no atomics): the sums are bit-identical across calls, graph replays,
// batch compositions and ranks.
#include <algorithm>

#include "common.cuh"
#include "cta_sum.cuh"
#include "resize_linear.cuh"

namespace b200 {

constexpr int kWarpThreads = 256;
constexpr int kWarpMaxBlocks = 1024;
constexpr int kWarpMaxSide = 32768;

static int warp_blocks(int64_t pixels) {
  const int64_t b = (pixels + kWarpThreads - 1) / kWarpThreads;
  return (int)(b < kWarpMaxBlocks ? b : kWarpMaxBlocks);
}

struct WarpPairDev {
  const void* f0;
  const void* f1;
  const float2* fwd;
  const float2* bwd;
  int H, W, bits, blocks;
  int64_t pix_off;          // first pixel of this pair in the per-pixel outputs
  int64_t part_off;         // first double of this pair's partials: [blocks] errors, then [blocks] counts
};
struct WarpBatch {
  WarpPairDev p[B200_WARP_MAX_PAIRS];
};

struct WarpResize {
  const float2* src[2];     // F, B (Hf, Wf)
  float2* dst[2];           // resized F, B (H, W) in the workspace
  int H, W, Hf, Wf;
  float sx, sy;
};
struct WarpResizeBatch {
  WarpResize r[B200_WARP_MAX_PAIRS];
};

__global__ void __launch_bounds__(256) warp_flow_resize_kernel(WarpResizeBatch b) {
  const WarpResize& r = b.r[blockIdx.y];
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (int64_t)r.H * r.W) return;
  const int y = (int)(p / r.W), x = (int)(p % r.W);
  const float2* src = r.src[blockIdx.z];
  const float vx = resize_sample<float>([&](int row, int col) { return src[(int64_t)row * r.Wf + col].x; }, r.Hf, r.Wf,
                                        r.H, r.W, y, x);
  const float vy = resize_sample<float>([&](int row, int col) { return src[(int64_t)row * r.Wf + col].y; }, r.Hf, r.Wf,
                                        r.H, r.W, y, x);
  r.dst[blockIdx.z][p] = make_float2(__fmul_rn(vx, r.sx), __fmul_rn(vy, r.sy));
}

// decoded value of channel c of pixel i: v / 255 or v / 65535 rounded to fp32, as a double
__device__ __forceinline__ double texel(const void* img, int bits, int64_t i) {
  const float v = bits == 8 ? __fdiv_rn((float)static_cast<const uint8_t*>(img)[i], 255.0f)
                            : __fdiv_rn((float)static_cast<const uint16_t*>(img)[i], 65535.0f);
  return (double)v;
}

// ((v00 (1 - ax) + v01 ax) (1 - ay) + (v10 (1 - ax) + v11 ax) ay)
__device__ __forceinline__ double lerp2(double v00, double v01, double v10, double v11, double ax, double bx, double ay,
                                        double by) {
  return add(mul(add(mul(v00, bx), mul(v01, ax)), by), mul(add(mul(v10, bx), mul(v11, ax)), ay));
}

__global__ void __launch_bounds__(kWarpThreads) warp_error_kernel(WarpBatch batch, double* __restrict__ partials,
                                                                  float* __restrict__ error, uint8_t* __restrict__ mask) {
  const WarpPairDev& pr = batch.p[blockIdx.y];
  if ((int)blockIdx.x >= pr.blocks) return;
  __shared__ double sh_e[kWarpThreads / 32], sh_n[kWarpThreads / 32];
  const int H = pr.H, W = pr.W;
  const int64_t pixels = (int64_t)H * W;
  double acc = 0.0, cnt = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * kWarpThreads + threadIdx.x; p < pixels; p += (int64_t)pr.blocks * kWarpThreads) {
    const int y = (int)(p / W), x = (int)(p % W);
    const float2 f = pr.fwd[p];
    const double fx = (double)f.x, fy = (double)f.y;
    const double qx = add((double)x, fx), qy = add((double)y, fy);
    float e = 0.f;
    bool m = false;
    if (qx >= 0.0 && qx <= (double)(W - 1) && qy >= 0.0 && qy <= (double)(H - 1)) {        // false for NaN too
      const int x0 = (int)floor(qx), y0 = (int)floor(qy);
      const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
      const double ax = __dsub_rn(qx, (double)x0), ay = __dsub_rn(qy, (double)y0);
      const double bx = __dsub_rn(1.0, ax), by = __dsub_rn(1.0, ay);
      const int64_t i00 = (int64_t)y0 * W + x0, i01 = (int64_t)y0 * W + x1;
      const int64_t i10 = (int64_t)y1 * W + x0, i11 = (int64_t)y1 * W + x1;
      const float2 b00 = pr.bwd[i00], b01 = pr.bwd[i01], b10 = pr.bwd[i10], b11 = pr.bwd[i11];
      const double wbx = lerp2(b00.x, b01.x, b10.x, b11.x, ax, bx, ay, by);
      const double wby = lerp2(b00.y, b01.y, b10.y, b11.y, ax, bx, ay, by);
      const double sx = add(fx, wbx), sy = add(fy, wby);
      const double lhs = add(mul(sx, sx), mul(sy, sy));
      const double rhs = add(mul(0.01, add(add(mul(fx, fx), mul(fy, fy)), add(mul(wbx, wbx), mul(wby, wby)))), 0.5);
      m = lhs <= rhs;
      double s = 0.0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double w = lerp2(texel(pr.f1, pr.bits, 3 * i00 + c), texel(pr.f1, pr.bits, 3 * i01 + c),
                               texel(pr.f1, pr.bits, 3 * i10 + c), texel(pr.f1, pr.bits, 3 * i11 + c), ax, bx, ay, by);
        const double d = __dsub_rn(texel(pr.f0, pr.bits, 3 * p + c), w);
        s = add(s, mul(d, d));
      }
      e = __double2float_rn(s);
    }
    if (m) {
      acc += (double)e;
      cnt += 1.0;
    }
    if (error) error[pr.pix_off + p] = e;
    if (mask) mask[pr.pix_off + p] = m ? 1 : 0;
  }
  acc = cta_sum<kWarpThreads>(acc, sh_e);
  cnt = cta_sum<kWarpThreads>(cnt, sh_n);
  if (threadIdx.x == 0) {
    partials[pr.part_off + blockIdx.x] = acc;
    partials[pr.part_off + pr.blocks + blockIdx.x] = cnt;
  }
}

__global__ void __launch_bounds__(kWarpThreads) warp_error_final_kernel(WarpBatch batch, const double* __restrict__ partials,
                                                                        double* __restrict__ sums) {
  const WarpPairDev& pr = batch.p[blockIdx.x];
  __shared__ double sh_e[kWarpThreads / 32], sh_n[kWarpThreads / 32];
  double acc = 0.0, cnt = 0.0;
  for (int i = threadIdx.x; i < pr.blocks; i += kWarpThreads) {
    acc += partials[pr.part_off + i];
    cnt += partials[pr.part_off + pr.blocks + i];
  }
  acc = cta_sum<kWarpThreads>(acc, sh_e);
  cnt = cta_sum<kWarpThreads>(cnt, sh_n);
  if (threadIdx.x == 0) {
    sums[2 * blockIdx.x] = acc;
    sums[2 * blockIdx.x + 1] = cnt;
  }
}

static bool needs_resize(const B200WarpPair& q) { return q.H != q.Hf || q.W != q.Wf; }

// Checks the descriptors and carves the workspace from byte 0: resized flows of the pairs that need them (F, then B,
// each 256-byte aligned), then the partials.  Returns the bytes needed, or -1 with the message set.
static int64_t plan_warp(const B200WarpPair* pairs, int n, WarpBatch* batch, WarpResizeBatch* rz, int* n_resize,
                         char* ws) {
  if (!pairs) {
    set_error("null pair table");
    return -1;
  }
  if (n < 1 || n > B200_WARP_MAX_PAIRS) {
    set_error("%d pairs: one call scores 1 to %d", n, B200_WARP_MAX_PAIRS);
    return -1;
  }
  int64_t off = 0, pix = 0;
  int k = 0;
  for (int i = 0; i < n; ++i) {
    const B200WarpPair& q = pairs[i];
    if (!q.frame0 || !q.frame1 || !q.fwd || !q.bwd) {
      set_error("pair %d: null pointer", i);
      return -1;
    }
    if (q.H <= 0 || q.W <= 0 || q.Hf <= 0 || q.Wf <= 0 || q.H > kWarpMaxSide || q.W > kWarpMaxSide ||
        q.Hf > kWarpMaxSide || q.Wf > kWarpMaxSide) {
      set_error("pair %d: frames %d x %d, flows %d x %d: each side must be in [1, %d]", i, q.H, q.W, q.Hf, q.Wf,
                kWarpMaxSide);
      return -1;
    }
    if (q.bits != 8 && q.bits != 16) {
      set_error("pair %d: pixels of %d bits; frames are uint8 (8) or uint16 (16)", i, q.bits);
      return -1;
    }
    if ((reinterpret_cast<uintptr_t>(q.fwd) & 7) || (reinterpret_cast<uintptr_t>(q.bwd) & 7) ||
        (q.bits == 16 && ((reinterpret_cast<uintptr_t>(q.frame0) & 1) || (reinterpret_cast<uintptr_t>(q.frame1) & 1)))) {
      set_error("pair %d: flows must be 8-byte aligned, 16-bit frames 2-byte aligned", i);
      return -1;
    }
    const int64_t hw = (int64_t)q.H * q.W;
    WarpPairDev& d = batch->p[i];
    d.f0 = q.frame0;
    d.f1 = q.frame1;
    d.fwd = reinterpret_cast<const float2*>(q.fwd);
    d.bwd = reinterpret_cast<const float2*>(q.bwd);
    d.H = q.H;
    d.W = q.W;
    d.bits = q.bits;
    d.blocks = warp_blocks(hw);
    d.pix_off = pix;
    pix += hw;
    if (needs_resize(q)) {
      WarpResize& r = rz->r[k++];
      r.src[0] = d.fwd;
      r.src[1] = d.bwd;
      for (int j = 0; j < 2; ++j) {
        r.dst[j] = reinterpret_cast<float2*>(reinterpret_cast<uintptr_t>(ws) + off);   // unused when ws is NULL
        off = round_up(off + hw * (int64_t)sizeof(float2), 256);
      }
      r.H = q.H; r.W = q.W; r.Hf = q.Hf; r.Wf = q.Wf;
      r.sx = (float)((double)q.W / (double)q.Wf);
      r.sy = (float)((double)q.H / (double)q.Hf);
      d.fwd = r.dst[0];
      d.bwd = r.dst[1];
    }
  }
  for (int i = 0; i < n; ++i) {
    batch->p[i].part_off = off / (int64_t)sizeof(double);
    off += 2 * (int64_t)batch->p[i].blocks * (int64_t)sizeof(double);
  }
  *n_resize = k;
  return off;
}

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_warp_error_workspace_bytes(const B200WarpPair* pairs_host, int32_t n) {
  WarpBatch batch;
  WarpResizeBatch rz;
  int k = 0;
  return plan_warp(pairs_host, n, &batch, &rz, &k, nullptr);
}

int b200_warp_error(const B200WarpPair* pairs_host, int32_t n, double* sums, float* error, uint8_t* mask, void* ws,
                    int64_t ws_bytes, void* stream) {
  B200_REQUIRE(sums && ws, "null pointer (sums and the workspace are required; error and mask may be NULL)");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 7) == 0, "workspace must be 8-byte aligned");
  WarpBatch batch;
  WarpResizeBatch rz;
  int k = 0;
  const int64_t need = plan_warp(pairs_host, n, &batch, &rz, &k, static_cast<char*>(ws));
  if (need < 0) return B200_ERR_INVALID;
  if (ws_bytes < need) {
    set_error("workspace too small: need %lld bytes", (long long)need);
    return B200_ERR_WORKSPACE;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (k > 0) {
    int64_t most = 0;
    for (int i = 0; i < k; ++i) most = std::max(most, (int64_t)rz.r[i].H * rz.r[i].W);
    warp_flow_resize_kernel<<<dim3((unsigned)((most + 255) / 256), k, 2), 256, 0, st>>>(rz);
    B200_CHECK_LAUNCH();
  }
  int grid = 0;
  for (int i = 0; i < n; ++i) grid = std::max(grid, batch.p[i].blocks);
  double* partials = reinterpret_cast<double*>(ws);
  warp_error_kernel<<<dim3(grid, n), kWarpThreads, 0, st>>>(batch, partials, error, mask);
  B200_CHECK_LAUNCH();
  warp_error_final_kernel<<<n, kWarpThreads, 0, st>>>(batch, partials, sums);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
