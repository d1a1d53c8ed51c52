// Float64 sum of squared differences between a rendered frame and that frame's resident pixel records — the numerator
// of the evaluation's per-frame PSNR (src/models/stage_1/evaluate.py:740-743) computed where the frame already is, so a
// frame-sharded evaluation needs no host copy of the video.
//
// The reduction order is a function of the frame size alone: a fixed grid of per-CTA partials (grid-stride over the
// pixels, then a shuffle / shared-memory tree), then one CTA that sums the partials in the same tree.  No atomics, so
// the result is bit-identical across calls, CUDA-graph replays, devices and ranks.
#include "atlas_internal.cuh"
#include "cta_sum.cuh"

namespace b200 {

constexpr int kSseThreads = 256;
constexpr int kSseMaxBlocks = 1024;

static int sse_blocks(int64_t pixels) {
  const int64_t b = (pixels + kSseThreads - 1) / kSseThreads;
  return (int)(b < kSseMaxBlocks ? b : kSseMaxBlocks);
}

__global__ void __launch_bounds__(kSseThreads) frame_sse_partial_kernel(const float* __restrict__ records,
                                                                         const float* __restrict__ rgb, int64_t pixels,
                                                                         double* __restrict__ partials) {
  __shared__ double sh[kSseThreads / 32];
  double acc = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * kSseThreads + threadIdx.x; p < pixels; p += (int64_t)gridDim.x * kSseThreads) {
    const float4 r = __ldg(reinterpret_cast<const float4*>(records + p * B200_RECORD_FLOATS));   // rgb in 0..2
    const double d0 = (double)__ldg(rgb + 3 * p) - (double)r.x;
    const double d1 = (double)__ldg(rgb + 3 * p + 1) - (double)r.y;
    const double d2 = (double)__ldg(rgb + 3 * p + 2) - (double)r.z;
    acc += d0 * d0;
    acc += d1 * d1;
    acc += d2 * d2;
  }
  acc = cta_sum<kSseThreads>(acc, sh);
  if (threadIdx.x == 0) partials[blockIdx.x] = acc;
}

__global__ void __launch_bounds__(kSseThreads) frame_sse_final_kernel(const double* __restrict__ partials, int n,
                                                                       double* __restrict__ out) {
  __shared__ double sh[kSseThreads / 32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += kSseThreads) acc += partials[i];
  acc = cta_sum<kSseThreads>(acc, sh);
  if (threadIdx.x == 0) *out = acc;
}

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_frame_sse_workspace_bytes(int32_t H, int32_t W) {
  if (H <= 0 || W <= 0) {
    set_error("frame size %d x %d out of range", H, W);
    return -1;
  }
  return (int64_t)sse_blocks((int64_t)H * W) * (int64_t)sizeof(double);
}

int b200_frame_sse(const B200Video* video, int32_t frame, const float* rgb, double* out, void* ws, int64_t ws_bytes,
                   void* stream) {
  B200_REQUIRE(video && video->records && rgb && out && ws, "null pointer");
  B200_REQUIRE(video->H > 0 && video->W > 0, "frame size %d x %d out of range", video->H, video->W);
  B200_REQUIRE(frame >= video->t_begin && frame < video->t_end, "frame %d is not resident (frames [%d, %d))", frame,
               video->t_begin, video->t_end);
  B200_REQUIRE((reinterpret_cast<uintptr_t>(video->records) & 15) == 0, "records must be 16-byte aligned");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 7) == 0, "workspace must be 8-byte aligned");
  const int64_t pixels = (int64_t)video->H * video->W;
  const int blocks = sse_blocks(pixels);
  if (ws_bytes < (int64_t)blocks * (int64_t)sizeof(double)) {
    set_error("workspace too small: need %lld bytes", (long long)blocks * (long long)sizeof(double));
    return B200_ERR_WORKSPACE;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  double* partials = reinterpret_cast<double*>(ws);
  const float* rec = video->records + (int64_t)(frame - video->t_begin) * pixels * B200_RECORD_FLOATS;
  frame_sse_partial_kernel<<<blocks, kSseThreads, 0, st>>>(rec, rgb, pixels, partials);
  B200_CHECK_LAUNCH();
  frame_sse_final_kernel<<<1, kSseThreads, 0, st>>>(partials, blocks, out);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
