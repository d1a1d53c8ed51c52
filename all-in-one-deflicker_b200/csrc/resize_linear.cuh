// One axis of cv2.resize(INTER_LINEAR) as OpenCV's own code computes it (imgproc resize.cpp; restated on the CPU in
// oracle/loader_oracle.py and oracle/stage2_io_oracle.py, pinned against cv2.resize): the sampling position of index d is
// fp32((d + 0.5) * (src / dst) - 0.5) with the product in float64, s = floor, weight = position - s in fp32, and the two
// taps are the source indices s and s + 1 clipped into the image.  The horizontal pass also zeroes the weight of a
// position outside [0, src - 1] (`clamp_weight`); the vertical pass does not, it only clips the row indices, so on an
// up-scale its border rows are S * (1 - w) + S * w, which is not always S.  Shared by the flow resize of the stage-1
// producer (producer.cu), the stage-2 frame kernels (stage2_io.cu) and the warping error's flow resize
// (warp_error.cu).
#pragma once

namespace b200 {

struct ResizeTap { int s0, s1; float w0, w1; };

__device__ __forceinline__ ResizeTap resize_tap(int d, int dst, int src, bool clamp_weight) {
  const double scale = (double)src / (double)dst;
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  ResizeTap t;
  if (clamp_weight) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= src - 1) { f = 0.f; s = src - 1; }
    t.s0 = s; t.s1 = min(s + 1, src - 1);
  } else {
    t.s0 = min(max(s, 0), src - 1); t.s1 = min(max(s + 1, 0), src - 1);
  }
  t.w1 = f; t.w0 = __fsub_rn(1.0f, f);
  return t;
}

// single IEEE operations in either arithmetic: the compiler must not contract a product and a sum into an fma
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }

// Bilinear sample of one channel at destination (y, x); `at(row, col)` reads the source in the arithmetic type T.
template <typename T, typename At>
__device__ __forceinline__ T resize_sample(At at, int h, int w, int H, int W, int y, int x) {
  if (h == H && w == W) return at(y, x);
  if (h == 2 * H && w == 2 * W)
    return mul(add(add(add(at(2 * y, 2 * x), at(2 * y, 2 * x + 1)), at(2 * y + 1, 2 * x)), at(2 * y + 1, 2 * x + 1)), (T)0.25);
  const ResizeTap tx = resize_tap(x, W, w, true), ty = resize_tap(y, H, h, false);
  const T r0 = add(mul(at(ty.s0, tx.s0), (T)tx.w0), mul(at(ty.s0, tx.s1), (T)tx.w1));
  const T r1 = add(mul(at(ty.s1, tx.s0), (T)tx.w0), mul(at(ty.s1, tx.s1), (T)tx.w1));
  return add(mul(r0, (T)ty.w0), mul(r1, (T)ty.w1));
}

}  // namespace b200
