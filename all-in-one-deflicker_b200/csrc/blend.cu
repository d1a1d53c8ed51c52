// Cross-fade of two renders of one frame (DESIGN §5): the frames two overlapping clips share are written as
// (1 - w) a + w b of the two atlases' renders, with w stepping linearly over the overlap.
//
// Per value the arithmetic is float64 with single IEEE operations (no fma contraction), rounded to fp32 once, so a
// numpy restatement in the same order reproduces every bit, and w = 0 / w = 1 return a / b exactly.  The 8-bit value
// is the truncation render_out_kernel (atlas_kernels.cu) and seg_compose_kernel (seg.cu) use, so a blended frame is
// quantised as a rendered one.  Memory-bound: 8 bytes read and up to 5 written per value.
#include <math.h>

#include "common.cuh"

namespace b200 {

constexpr int kBlendThreads = 256;
constexpr int kBlendMaxBlocks = 132 * 16;

__global__ void __launch_bounds__(kBlendThreads) blend_frames_kernel(const float* __restrict__ a,
                                                                     const float* __restrict__ b, int64_t n, double w,
                                                                     double wa, float* __restrict__ out,
                                                                     uint8_t* __restrict__ u8) {
  for (int64_t i = (int64_t)blockIdx.x * kBlendThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlendThreads) {
    const double v = __dadd_rn(__dmul_rn(wa, (double)a[i]), __dmul_rn(w, (double)b[i]));
    const float o = __double2float_rn(v);
    if (out) out[i] = o;
    if (u8) u8[i] = (uint8_t)(int)__dmul_rn((double)o, 255.0);
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_blend_frames(const float* a, const float* b, int64_t n, double w, float* out, uint8_t* u8, void* stream) {
  B200_REQUIRE(a && b, "null input (a and b are required)");
  B200_REQUIRE(out || u8, "out and u8 are both NULL: nothing to write");
  B200_REQUIRE(n >= 1, "%lld values: n must be >= 1", (long long)n);
  B200_REQUIRE(isfinite(w) && w >= 0.0 && w <= 1.0, "weight %g: w must be finite and in [0, 1]", w);
  const int64_t need = (n + kBlendThreads - 1) / kBlendThreads;
  const int blocks = (int)(need < kBlendMaxBlocks ? need : kBlendMaxBlocks);
  blend_frames_kernel<<<blocks, kBlendThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a, b, n, w, 1.0 - w, out,
                                                                                            u8);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
