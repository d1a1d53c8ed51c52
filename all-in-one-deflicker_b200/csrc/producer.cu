// Device-side input producer of the stage-1 loop (SURVEY.md §8f rank 1): what the reference's
// load_input_data_single (src/models/stage_1/unwrap_utils.py:105-163) computes per frame and per frame pair,
// written straight into the frame-major pixel records and the validity bitmaps of B200Video — the eight
// (H, W, ., T) host tensors of the reference (1.6 GB at 80 x 432 x 768) are never built.
//
//   producer_frame_kernel       rgb + forward differences of one decoded frame            unwrap_utils.py:131-133
//   producer_resize_kernel      resize_flow: cv2.resize(INTER_LINEAR) + the reference's swapped scale factors
//                               (x by newh/oldh, y by neww/oldw)                            unwrap_utils.py:33-38
//   producer_consistency_kernel compute_consistency(flow_a, flow_b) < 1.0: cv2.remap of flow_b at p + flow_a
//                               (bilinear, 1/32-pixel coordinate grid, zero border), |flow_a + warped|   :10-23,148-149
// The arithmetic is the bit-exact restatement pinned against OpenCV in oracle/loader_oracle.py
// (tests/test_loader_oracle.py); tests/test_producer_gpu.py compares records and bitmaps with the reference's tensors.
// Decoding image files and the float64 frame resize stay on the host, one frame at a time.
#include "common.cuh"
#include "resize_linear.cuh"

namespace b200 {

__global__ void producer_frame_kernel(const float* __restrict__ frame, int H, int W, float* __restrict__ rec) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (int64_t)H * W) return;
  const int y = (int)(p / W), x = (int)(p % W);
  float v[9];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float a = frame[p * 3 + c];
    v[c] = a;
    v[3 + c] = x + 1 < W ? __fsub_rn(frame[(p + 1) * 3 + c], a) : 0.f;          // dx, zero in the last column
    v[6 + c] = y + 1 < H ? __fsub_rn(frame[(p + W) * 3 + c], a) : 0.f;          // dy, zero in the last row
  }
  float4* dst = reinterpret_cast<float4*>(rec + p * B200_RECORD_FLOATS);
  dst[0] = make_float4(v[0], v[1], v[2], v[3]);
  dst[1] = make_float4(v[4], v[5], v[6], v[7]);
  rec[p * B200_RECORD_FLOATS + 8] = v[8];
}

// dst (H, W, 2) <- src (h, w, 2), H <= h and W <= w; then the reference's scale factors
__global__ void producer_resize_kernel(const float2* __restrict__ src, int h, int w, float2* __restrict__ dst, int H,
                                       int W, float sx, float sy) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (int64_t)H * W) return;
  const int y = (int)(p / W), x = (int)(p % W);
  float2 o;
  if (h == 2 * H && w == 2 * W) {                       // OpenCV's area-fast path for exactly half size
    const float2 a = src[(int64_t)(2 * y) * w + 2 * x], b = src[(int64_t)(2 * y) * w + 2 * x + 1];
    const float2 c = src[(int64_t)(2 * y + 1) * w + 2 * x], d = src[(int64_t)(2 * y + 1) * w + 2 * x + 1];
    o.x = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(a.x, b.x), c.x), d.x), 0.25f);
    o.y = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(a.y, b.y), c.y), d.y), 0.25f);
  } else {
    const ResizeTap tx = resize_tap(x, W, w, true), ty = resize_tap(y, H, h, false);
    const float2 a0 = src[(int64_t)ty.s0 * w + tx.s0], a1 = src[(int64_t)ty.s0 * w + tx.s1];
    const float2 b0 = src[(int64_t)ty.s1 * w + tx.s0], b1 = src[(int64_t)ty.s1 * w + tx.s1];
    const float r0x = __fadd_rn(__fmul_rn(a0.x, tx.w0), __fmul_rn(a1.x, tx.w1));
    const float r0y = __fadd_rn(__fmul_rn(a0.y, tx.w0), __fmul_rn(a1.y, tx.w1));
    const float r1x = __fadd_rn(__fmul_rn(b0.x, tx.w0), __fmul_rn(b1.x, tx.w1));
    const float r1y = __fadd_rn(__fmul_rn(b0.y, tx.w0), __fmul_rn(b1.y, tx.w1));
    o.x = __fadd_rn(__fmul_rn(r0x, ty.w0), __fmul_rn(r1x, ty.w1));
    o.y = __fadd_rn(__fmul_rn(r0y, ty.w0), __fmul_rn(r1y, ty.w1));
  }
  o.x = __fmul_rn(o.x, sx);
  o.y = __fmul_rn(o.y, sy);
  dst[p] = o;
}

__device__ __forceinline__ float2 remap_tap(const float2* img, int H, int W, int y, int x) {
  if (x < 0 || x >= W || y < 0 || y >= H) return make_float2(0.f, 0.f);
  return img[(int64_t)y * W + x];
}

// mask(p) = | fa(p) + remap(fb)(p + fa(p)) | < 1, written with the flow fa itself into the record slot `flow_off` /
// `mask_off` of frame `rec` (nullptr: frame not resident here) and into the whole-video bitmap at pixel-table offset `n0`
__global__ void producer_consistency_kernel(const float2* __restrict__ fa, const float2* __restrict__ fb, int H, int W,
                                            float* __restrict__ rec, int flow_off, int mask_off,
                                            uint32_t* __restrict__ bits, int64_t n0, int filter) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t HW = (int64_t)H * W;
  bool valid = false;
  if (p < HW) {
    const int y = (int)(p / W), x = (int)(p % W);
    const float2 f = fa[p];
    valid = true;
    if (filter) {
      const float mx = __fadd_rn(f.x, (float)x), my = __fadd_rn(f.y, (float)y);
      // cv2.remap: coordinates on a 1/32-pixel grid, round half to even (the products by 32 are exact)
      const int qx = __float2int_rn(mx * 32.0f), qy = __float2int_rn(my * 32.0f);
      const int ix = qx >> 5, iy = qy >> 5;
      const float wx = (float)(qx & 31) * 0.03125f, wy = (float)(qy & 31) * 0.03125f;
      const float w_nw = __fmul_rn(__fsub_rn(1.f, wy), __fsub_rn(1.f, wx)), w_ne = __fmul_rn(__fsub_rn(1.f, wy), wx);
      const float w_sw = __fmul_rn(wy, __fsub_rn(1.f, wx)), w_se = __fmul_rn(wy, wx);
      const float2 nw = remap_tap(fb, H, W, iy, ix), ne = remap_tap(fb, H, W, iy, ix + 1);
      const float2 sw = remap_tap(fb, H, W, iy + 1, ix), se = remap_tap(fb, H, W, iy + 1, ix + 1);
      const float wpx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(nw.x, w_nw), __fmul_rn(ne.x, w_ne)), __fmul_rn(sw.x, w_sw)),
                                  __fmul_rn(se.x, w_se));
      const float wpy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(nw.y, w_nw), __fmul_rn(ne.y, w_ne)), __fmul_rn(sw.y, w_sw)),
                                  __fmul_rn(se.y, w_se));
      const float dx = __fadd_rn(f.x, wpx), dy = __fadd_rn(f.y, wpy);
      const float err = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
      valid = err < 1.0f;
    }
    if (rec) {
      float* r = rec + p * B200_RECORD_FLOATS;
      r[flow_off] = f.x; r[flow_off + 1] = f.y;
      r[mask_off] = valid ? 1.f : 0.f;
    }
  }
  // bitmap bit n0 + p; a warp's 32 pixels may straddle two words
  const uint32_t ballot = __ballot_sync(0xffffffffu, valid);
  if ((threadIdx.x & 31) == 0 && ballot) {
    const int64_t n = n0 + p;                       // p of lane 0
    const int sh = (int)(n & 31);
    atomicOr(bits + (n >> 5), ballot << sh);
    if (sh) atomicOr(bits + (n >> 5) + 1, ballot >> (32 - sh));
  }
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_producer_frame(const float* frame, int32_t H, int32_t W, float* frame_records, void* stream) {
  B200_REQUIRE(frame && frame_records && H > 0 && W > 0, "bad frame arguments");
  const int64_t n = (int64_t)H * W;
  producer_frame_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(frame, H, W,
                                                                                                           frame_records);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int64_t b200_producer_scratch_floats(int32_t H, int32_t W) { return (int64_t)H * W * 4; }

int b200_producer_flow_pair(const float* flow12, const float* flow21, int32_t h, int32_t w, int32_t H, int32_t W,
                            int32_t T, int32_t t_begin, int32_t t_end, float* records, uint32_t* mask_fwd_bits,
                            uint32_t* mask_bwd_bits, int32_t first_frame, int32_t filter, float* scratch, void* stream) {
  B200_REQUIRE(flow12 && flow21 && scratch && mask_fwd_bits && mask_bwd_bits, "null pointer");
  B200_REQUIRE(H > 0 && W > 0 && first_frame >= 0 && first_frame + 1 < T && t_begin >= 0 && t_end <= T &&
               t_begin <= t_end, "bad frame pair %d", first_frame);
  B200_REQUIRE(h >= H && w >= W, "the device resize covers down-scaling only (flow %dx%d -> %dx%d): resize on the host",
               h, w, H, W);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t HW = (int64_t)H * W;
  const unsigned blocks = (unsigned)((HW + 255) / 256);
  const float2* f12 = reinterpret_cast<const float2*>(flow12);
  const float2* f21 = reinterpret_cast<const float2*>(flow21);
  if (h != H || w != W) {
    // resize_flow: x scaled by newh/oldh and y by neww/oldw, as the reference has it (unwrap_utils.py:36-37)
    const float sx = (float)((double)H / (double)h), sy = (float)((double)W / (double)w);
    float2* r12 = reinterpret_cast<float2*>(scratch);
    float2* r21 = r12 + HW;
    producer_resize_kernel<<<blocks, 256, 0, st>>>(f12, h, w, r12, H, W, sx, sy);
    B200_CHECK_LAUNCH();
    producer_resize_kernel<<<blocks, 256, 0, st>>>(f21, h, w, r21, H, W, sx, sy);
    B200_CHECK_LAUNCH();
    f12 = r12; f21 = r21;
  }
  const int i = first_frame, j = first_frame + 1;
  float* rec_i = (records && i >= t_begin && i < t_end) ? records + (int64_t)(i - t_begin) * HW * B200_RECORD_FLOATS : nullptr;
  float* rec_j = (records && j >= t_begin && j < t_end) ? records + (int64_t)(j - t_begin) * HW * B200_RECORD_FLOATS : nullptr;
  // forward: flow i -> j stored with frame i;  backward: flow j -> i stored with frame j (unwrap_utils.py:151-158)
  producer_consistency_kernel<<<blocks, 256, 0, st>>>(f12, f21, H, W, rec_i, 9, 13, mask_fwd_bits, (int64_t)i * HW, filter);
  B200_CHECK_LAUNCH();
  producer_consistency_kernel<<<blocks, 256, 0, st>>>(f21, f12, H, W, rec_j, 11, 14, mask_bwd_bits, (int64_t)j * HW, filter);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
