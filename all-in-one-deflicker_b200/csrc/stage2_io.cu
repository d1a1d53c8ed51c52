// Frame plumbing of stage 2 on the device (SURVEY.md §3.5): what the reference's script does on the host around the two
// networks, per frame, from 8-bit images to 8-bit images.
//
//   stage2_pack_kernel  load_image x2 + InputPadder.pad + torch.cat (src/models/utils.py, neural_filter_and_refinement.py):
//                       content / 255 and the atlas frame / 255 resized to the content's size, both replicate-padded to
//                       multiples of 32, as one [1, 6, Hp, Wp] fp32 tensor
//   stage2_emit_kernel  cv2.resize(tensor2img(t), org_size) + save_img's clip(v * 255, 0, 255).astype(uint8) and RGB -> BGR,
//                       written into a panel of a caller-owned 8-bit image
//
// The resize is OpenCV's own INTER_LINEAR code path, restated in oracle/stage2_io_oracle.py (resize_linear_f64 /
// resize_linear_f32) and pinned there against cv2.resize: taps and weights in fp32 (resize_linear.cuh), horizontal pass then
// vertical pass, products and sums rounded separately; equal sizes copy, exactly half size in both dimensions is the 2x2
// mean (((a + b) + c) + d) * 0.25.  load_image divides and resizes in float64 and rounds to fp32 once; tensor2img's
// resize is fp32 throughout.
#include "common.cuh"
#include "resize_linear.cuh"

namespace b200 {

// 8-bit HWC image with 1, 3 or 4 channels read as the reference reads it: grey repeated, a 4th channel dropped
struct U8Image {
  const uint8_t* p; int h, w, c;
  __device__ __forceinline__ double at(int y, int x, int ch) const {
    return (double)p[((int64_t)y * w + x) * c + (c == 1 ? 0 : ch)] / 255.0;
  }
};

__global__ void stage2_pack_kernel(U8Image content, U8Image atlas, float* __restrict__ out, int Hp, int Wp) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= Wp) return;
  const int pad_left = (Wp - content.w) / 2;
  const int cy = min(y, content.h - 1), cx = min(max(x - pad_left, 0), content.w - 1);      // replicate padding
  const int64_t plane = (int64_t)Hp * Wp, o = (int64_t)y * Wp + x;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    out[ch * plane + o] = (float)content.at(cy, cx, ch);
    out[(3 + ch) * plane + o] = (float)resize_sample<double>([&](int r, int c) { return atlas.at(r, c, ch); }, atlas.h,
                                                             atlas.w, content.h, content.w, cy, cx);
  }
}

// NaN becomes 0 (fmaxf returns its other operand); numpy's cast of NaN to uint8 is platform-defined and not reproduced.
__global__ void stage2_emit_kernel(const float* __restrict__ src, int64_t plane, int Hp, int Wp, uint8_t* __restrict__ dst,
                                   int64_t row_stride, int H, int W) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= W) return;
  uint8_t* px = dst + (int64_t)y * row_stride + 3 * x;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float* s = src + ch * plane;
    const float v = resize_sample<float>([&](int r, int c) { return s[(int64_t)r * Wp + c]; }, Hp, Wp, H, W, y, x);
    px[2 - ch] = (uint8_t)(int)fminf(fmaxf(__fmul_rn(v, 255.0f), 0.f), 255.f);              // truncation; RGB -> BGR
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_stage2_pack_input(const uint8_t* content, int32_t Hc, int32_t Wc, int32_t Cc, const uint8_t* atlas, int32_t Hs,
                           int32_t Ws, int32_t Cs, float* out, int32_t Hp, int32_t Wp, void* stream) {
  B200_REQUIRE(content && atlas && out, "null pointer");
  B200_REQUIRE(Hc > 0 && Wc > 0 && Hs > 0 && Ws > 0, "bad image size %dx%d / %dx%d", Hc, Wc, Hs, Ws);
  B200_REQUIRE((Cc == 1 || Cc == 3 || Cc == 4) && (Cs == 1 || Cs == 3 || Cs == 4),
               "images have 1, 3 or 4 channels (got %d and %d)", Cc, Cs);
  B200_REQUIRE(Hp == (Hc + 31) / 32 * 32 && Wp == (Wc + 31) / 32 * 32 && Hp <= 65535,
               "padded size %dx%d is not %dx%d rounded up to multiples of 32", Hp, Wp, Hc, Wc);
  const U8Image c{content, Hc, Wc, Cc}, a{atlas, Hs, Ws, Cs};
  stage2_pack_kernel<<<dim3((Wp + 127) / 128, Hp), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(c, a, out, Hp, Wp);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_stage2_emit(const float* src, int64_t plane_stride, int32_t Hp, int32_t Wp, uint8_t* dst, int64_t dst_offset,
                     int64_t dst_row_stride, int32_t H, int32_t W, void* stream) {
  B200_REQUIRE(src && dst, "null pointer");
  B200_REQUIRE(Hp > 0 && Wp > 0 && H > 0 && W > 0 && H <= 65535, "bad size %dx%d -> %dx%d", Hp, Wp, H, W);
  B200_REQUIRE(plane_stride >= (int64_t)Hp * Wp, "channel stride %lld is smaller than a %dx%d plane",
               (long long)plane_stride, Hp, Wp);
  B200_REQUIRE(dst_offset >= 0 && dst_row_stride >= 3 * (int64_t)W, "row stride %lld cannot hold %d BGR pixels",
               (long long)dst_row_stride, W);
  stage2_emit_kernel<<<dim3((W + 127) / 128, H), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, plane_stride, Hp, Wp, dst + dst_offset, dst_row_stride, H, W);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
