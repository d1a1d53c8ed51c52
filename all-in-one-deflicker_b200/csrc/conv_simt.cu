// fp32 implicit-GEMM convolution and the small image operators the RAFT update block and the stage-2
// networks need (NCHW tensors, the reference's layouts).
//
// Restates, on the reference side:
//   nn.Conv2d (+ bias, ReLU / LeakyReLU(0.2) / sigmoid / tanh), nn.ReflectionPad2d, nn.Upsample(nearest)
//     src/models/network_local.py:118-188, src/models/network_filter.py:8-107,
//     src/models/stage_1/core/update.py:6-136
//   nn.MaxPool2d(2,2), nn.Upsample(scale 2, bilinear, align_corners=True)   network_filter.py:13-26
//   SepConvGRU / ConvLSTM gating                                             update.py:33-60, network_local.py:38-53
//   convex 8x flow upsampling                                                core/raft.py:76-87
#include "common.cuh"

namespace b200 {

constexpr int CBI = 128, CBJ = 128, CBR = 16, CPAD = 132, CONV_THREADS = 256;

struct ConvArgs {
  B200ConvDesc d;
  const float* x; const float* w; const float* bias; const float* res; float* y;
  int OH, OW, R;            // output size, reduction length Cin*KH*KW
  int64_t pixels;           // N*OH*OW
};

__device__ __forceinline__ float conv_act(float v, int act) {
  switch (act) {
    case 1: return fmaxf(v, 0.f);
    case 2: return v > 0.f ? v : 0.2f * v;
    case 3: return 1.0f / (1.0f + expf(-v));
    case 4: return tanhf(v);
    default: return v;
  }
}

__device__ __forceinline__ int reflect_idx(int i, int n) {       // nn.ReflectionPad2d index map
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// C[pixel][cout] = sum_r X(pixel, r) * W[cout][r]; pixel tile on I, cout tile on J
__global__ void __launch_bounds__(CONV_THREADS, 2) conv2d_kernel(ConvArgs a) {
  __shared__ __align__(16) float Ps[2][CBR][CPAD];
  __shared__ __align__(16) float Qs[2][CBR][CPAD];
  const B200ConvDesc& d = a.d;
  const int tid = threadIdx.x;
  const int64_t i0 = (int64_t)blockIdx.x * CBI;
  const int j0 = blockIdx.y * CBJ;
  const int ty = tid / 16, tx = tid % 16;
  // this thread gathers 4 consecutive pixels (o4..o4+3) for rows r = tid/32 + 8*it of every reduction tile
  const int o4 = (tid % 32) * 4;
  int pn[4], py[4], px[4];
  const int HU = d.H * d.upsample, WU = d.W * d.upsample;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int64_t p = i0 + o4 + q;
    if (p < a.pixels) {
      const int ox = (int)(p % a.OW);
      const int oy = (int)((p / a.OW) % a.OH);
      pn[q] = (int)(p / ((int64_t)a.OW * a.OH));
      py[q] = oy * d.stride - d.pad_h;
      px[q] = ox * d.stride - d.pad_w;
    } else { pn[q] = -1; py[q] = px[q] = 0; }
  }
  const int KHW = d.KH * d.KW;
  auto load_tiles = [&](int buf, int r0) {
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int r = tid / 32 + 8 * it;
      const int gr = r0 + r;
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gr < a.R) {
        const int ci = gr / KHW, kk = gr % KHW, ky = kk / d.KW, kx = kk % d.KW;
        float v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          v[q] = 0.f;
          if (pn[q] >= 0) {
            int iy = py[q] + ky, ix = px[q] + kx;
            bool ok = true;
            if (d.pad_mode == 1) { iy = reflect_idx(iy, HU); ix = reflect_idx(ix, WU); }
            else ok = (iy >= 0 && iy < HU && ix >= 0 && ix < WU);
            if (ok) {
              if (d.upsample > 1) { iy /= d.upsample; ix /= d.upsample; }
              v[q] = __ldg(a.x + (((int64_t)pn[q] * d.in_c_total + d.in_c_off + ci) * d.H + iy) * d.W + ix);
            }
          }
        }
        t = make_float4(v[0], v[1], v[2], v[3]);
      }
      *reinterpret_cast<float4*>(&Ps[buf][r][o4]) = t;
    }
    // weights: W[cout][r], r contiguous: thread loads 4 consecutive r of one cout
#pragma unroll
    for (int it = 0; it < (CBJ * CBR / 4) / CONV_THREADS; ++it) {
      const int e = tid + it * CONV_THREADS;
      const int o = e / (CBR / 4), r4 = (e % (CBR / 4)) * 4;
      const int go = j0 + o, gr = r0 + r4;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (go < d.Cout) {
        const float* src = a.w + (int64_t)go * a.R + gr;
#pragma unroll
        for (int q = 0; q < 4; ++q) if (gr + q < a.R) v[q] = __ldg(src + q);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) Qs[buf][r4 + q][o] = v[q];
    }
  };
  float acc[8][8];
#pragma unroll
  for (int u = 0; u < 8; ++u)
#pragma unroll
    for (int v = 0; v < 8; ++v) acc[u][v] = 0.f;
  int buf = 0;
  load_tiles(0, 0);
  __syncthreads();
  for (int r0 = 0; r0 < a.R; r0 += CBR) {
    if (r0 + CBR < a.R) load_tiles(buf ^ 1, r0 + CBR);
#pragma unroll
    for (int r = 0; r < CBR; ++r) {
      const float4 p0 = *reinterpret_cast<const float4*>(&Ps[buf][r][ty * 8]);
      const float4 p1 = *reinterpret_cast<const float4*>(&Ps[buf][r][ty * 8 + 4]);
      const float4 q0 = *reinterpret_cast<const float4*>(&Qs[buf][r][tx * 8]);
      const float4 q1 = *reinterpret_cast<const float4*>(&Qs[buf][r][tx * 8 + 4]);
      const float p[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
      const float q[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
      for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int v = 0; v < 8; ++v) acc[u][v] = fmaf(p[u], q[v], acc[u][v]);
    }
    __syncthreads();
    buf ^= 1;
  }
  const int64_t plane = (int64_t)a.OH * a.OW;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int64_t p = i0 + ty * 8 + u;
    if (p >= a.pixels) continue;
    const int64_t n = p / plane, sp = p % plane;
#pragma unroll
    for (int v = 0; v < 8; ++v) {
      const int j = j0 + tx * 8 + v;
      if (j >= d.Cout) continue;
      float val = acc[u][v];
      if (a.bias) val += a.bias[j];
      val = conv_act(val, d.act) * d.out_scale;
      if (a.res) val += a.res[(n * d.res_c_total + d.res_c_off + j) * plane + sp];
      a.y[(n * d.out_c_total + d.out_c_off + j) * plane + sp] = val;
    }
  }
}

// ------------------------------------------------------------------------------------------- pooling etc.
__global__ void maxpool2_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t planes, int H, int W) {
  const int OH = H / 2, OW = W / 2;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= planes * OH * OW) return;
  const int ox = (int)(i % OW), oy = (int)((i / OW) % OH);
  const int64_t pl = i / ((int64_t)OW * OH);
  const float* s = x + (pl * H + 2 * oy) * W + 2 * ox;
  y[i] = fmaxf(fmaxf(s[0], s[1]), fmaxf(s[W], s[W + 1]));
}

// nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True) into a channel slice of y
__global__ void upsample_bilinear2_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int C, int H,
                                          int W, int out_c_total, int out_c_off) {
  const int OH = 2 * H, OW = 2 * W;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)N * C * OH * OW) return;
  const int ox = (int)(i % OW), oy = (int)((i / OW) % OH);
  const int c = (int)((i / ((int64_t)OW * OH)) % C), n = (int)(i / ((int64_t)OW * OH * C));
  // ATen area_pixel_compute_source_index(align_corners=True): src = dst * (in-1)/(out-1)
  const float sh = OH > 1 ? (float)(H - 1) / (float)(OH - 1) : 0.f;
  const float sw = OW > 1 ? (float)(W - 1) / (float)(OW - 1) : 0.f;
  const float fy = sh * oy, fx = sw * ox;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
  const float ly = fy - y0, lx = fx - x0;
  const float* s = x + ((int64_t)n * C + c) * H * W;
  const float v = (1.f - ly) * ((1.f - lx) * s[y0 * W + x0] + lx * s[y0 * W + x1]) +
                  ly * ((1.f - lx) * s[y1 * W + x0] + lx * s[y1 * W + x1]);
  y[(((int64_t)n * out_c_total + out_c_off + c) * OH + oy) * OW + ox] = v;
}

// GRU gating.  mode 0: rh = sigmoid-activated r * h written into channels [0,C) of a concat buffer
//              mode 1: h_new = (1 - z) * h + z * q
__global__ void gru_gate_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c,
                                float* __restrict__ out, int64_t n_per_sample, int out_stride, int mode, int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t n = i / n_per_sample, k = i % n_per_sample;
  float v;
  if (mode == 0) v = a[i] * b[i];
  else v = (1.f - a[i]) * b[i] + a[i] * c[i];
  out[n * out_stride + k] = v;
}

// ConvLSTM cell (network_local.py:18-53): gates [N][4C][H][W] (pre-activation, chunk(4, 1) order in, remember, out,
// cell) -> cell = sigmoid(r) * prev_cell + sigmoid(i) * tanh(g), hidden = sigmoid(o) * tanh(cell).
// prev_cell == nullptr is prev_state=None: cell = sigmoid(i) * tanh(g).  The same expressions as the fused epilogue of
// convlstm_tma_kernel (conv_tma.cu).
__global__ void convlstm_cell_kernel(const float* __restrict__ gates, const float* __restrict__ prev_cell,
                                     float* __restrict__ hidden, float* __restrict__ cell, int C, int64_t plane,
                                     int64_t total) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t sp = i % plane, c = (i / plane) % C, n = i / (plane * C);
  const float* g = gates + n * 4 * C * plane;
  const float in_g = 1.f / (1.f + expf(-g[(c)*plane + sp]));
  const float out_g = 1.f / (1.f + expf(-g[(2 * C + c) * plane + sp]));
  const float cell_g = tanhf(g[(3 * C + c) * plane + sp]);
  float cl;
  if (prev_cell) {                                  // torch: (remember * prev) + (in * cell_gate), each rounded
    const float rem_g = 1.f / (1.f + expf(-g[(C + c) * plane + sp]));
    cl = __fadd_rn(__fmul_rn(rem_g, prev_cell[i]), __fmul_rn(in_g, cell_g));
  } else {
    cl = in_g * cell_g;                             // remember_gate * 0 + in_gate * cell_gate
  }
  hidden[i] = out_g * tanhf(cl);
  if (cell) cell[i] = cl;
}

// RAFT convex upsampling (core/raft.py:76-87): flow [N][2][H][W], mask [N][576][H][W] -> [N][2][8H][8W]
__global__ void convex_upsample_kernel(const float* __restrict__ flow, const float* __restrict__ mask,
                                       float* __restrict__ out, int N, int H, int W) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;       // over N*H*W*64 (fine positions)
  if (i >= (int64_t)N * H * W * 64) return;
  const int sub = (int)(i % 64), x = (int)((i / 64) % W), y = (int)((i / (64 * W)) % H), n = (int)(i / ((int64_t)64 * W * H));
  const int64_t plane = (int64_t)H * W;
  const float* m = mask + (int64_t)n * 576 * plane + (int64_t)y * W + x;
  float w[9], mx = -1e30f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { w[k] = m[(int64_t)(k * 64 + sub) * plane]; mx = fmaxf(mx, w[k]); }
  float den = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { w[k] = expf(w[k] - mx); den += w[k]; }
  const int sy = sub / 8, sx = sub % 8;
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;                    // F.unfold(…, [3,3], padding=1)
      const float f = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? 8.f * flow[((int64_t)n * 2 + c) * plane + (int64_t)yy * W + xx] : 0.f;
      acc += (w[k] / den) * f;
    }
    out[(((int64_t)n * 2 + c) * (8 * H) + (8 * y + sy)) * (8 * W) + 8 * x + sx] = acc;
  }
}

// nn.InstanceNorm2d (affine=False, eps) over each (n, c) plane, optional ReLU; one 1024-thread block per plane,
// float4 accesses when the plane size allows.  Two passes (mean, then centred variance) like ATen's
// batch_norm statistics; the plane is re-read from L2.
__device__ __forceinline__ float block_sum_1024(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                                       // red[] may still be read from the previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) {
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) red[32] = t;
  }
  __syncthreads();
  return red[32];
}

__global__ void __launch_bounds__(1024) instance_norm_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t hw,
                                                             float eps, int relu) {
  const float* s = x + (int64_t)blockIdx.x * hw;
  float* d = y + (int64_t)blockIdx.x * hw;
  __shared__ float red[33];
  const bool vec = (hw & 3) == 0;
  const int64_t nv = vec ? hw >> 2 : 0;
  const float4* s4 = reinterpret_cast<const float4*>(s);
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < nv; i += blockDim.x) { const float4 v = s4[i]; acc += (v.x + v.y) + (v.z + v.w); }
  for (int64_t i = nv * 4 + threadIdx.x; i < hw; i += blockDim.x) acc += s[i];
  const float mean = block_sum_1024(acc, red) / (float)hw;
  acc = 0.f;
  for (int64_t i = threadIdx.x; i < nv; i += blockDim.x) {
    const float4 v = s4[i];
    const float a = v.x - mean, b = v.y - mean, c = v.z - mean, e = v.w - mean;
    acc += (a * a + b * b) + (c * c + e * e);
  }
  for (int64_t i = nv * 4 + threadIdx.x; i < hw; i += blockDim.x) { const float c = s[i] - mean; acc += c * c; }
  const float inv = rsqrtf(block_sum_1024(acc, red) / (float)hw + eps);
  float4* d4 = reinterpret_cast<float4*>(d);
  for (int64_t i = threadIdx.x; i < nv; i += blockDim.x) {
    float4 v = s4[i];
    v.x = (v.x - mean) * inv; v.y = (v.y - mean) * inv; v.z = (v.z - mean) * inv; v.w = (v.w - mean) * inv;
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    d4[i] = v;
  }
  for (int64_t i = nv * 4 + threadIdx.x; i < hw; i += blockDim.x) {
    const float v = (s[i] - mean) * inv;
    d[i] = relu ? fmaxf(v, 0.f) : v;
  }
}

__global__ void add_relu_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = fmaxf(a[i] + b[i], 0.f);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_instance_norm(const float* x, float* y, int64_t planes, int64_t hw, float eps, int32_t relu, void* stream) {
  B200_REQUIRE(x && y && planes > 0 && hw > 0, "bad arguments");
  instance_norm_kernel<<<(unsigned)planes, 1024, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, y, hw, eps, relu);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_add_relu(const float* a, const float* b, float* out, int64_t n, void* stream) {
  B200_REQUIRE(a && b && out && n > 0, "bad arguments");
  add_relu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a, b, out, n);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_conv2d(const B200ConvDesc* d, const float* x, const float* w, const float* bias, const float* residual,
                float* y, void* stream) {
  B200_REQUIRE(d && d->upsample_mode == 0, "bilinear upsampling is fused only by b200_conv2d_tma_chain");
  B200_REQUIRE(d && x && w && y, "null pointer");
  B200_REQUIRE(d->N > 0 && d->Cin > 0 && d->H > 0 && d->W > 0 && d->Cout > 0 && d->KH > 0 && d->KW > 0 && d->stride > 0 &&
               (d->upsample == 1 || d->upsample == 2) && (d->pad_mode == 0 || d->pad_mode == 1) && d->act >= 0 && d->act <= 4,
               "invalid convolution descriptor");
  B200_REQUIRE(d->in_c_off >= 0 && d->in_c_off + d->Cin <= d->in_c_total && d->out_c_off >= 0 &&
               d->out_c_off + d->Cout <= d->out_c_total, "channel slice out of range");
  const int HU = d->H * d->upsample, WU = d->W * d->upsample;
  B200_REQUIRE(d->pad_mode == 0 || (d->pad_h < HU && d->pad_w < WU), "reflection padding larger than the input");
  ConvArgs a{};
  a.d = *d; a.x = x; a.w = w; a.bias = bias; a.res = residual; a.y = y;
  a.OH = (HU + 2 * d->pad_h - d->KH) / d->stride + 1;
  a.OW = (WU + 2 * d->pad_w - d->KW) / d->stride + 1;
  B200_REQUIRE(a.OH > 0 && a.OW > 0, "empty output");
  a.R = d->Cin * d->KH * d->KW;
  a.pixels = (int64_t)d->N * a.OH * a.OW;
  if (residual) B200_REQUIRE(d->res_c_off >= 0 && d->res_c_off + d->Cout <= d->res_c_total, "residual slice out of range");
  dim3 grid((unsigned)((a.pixels + CBI - 1) / CBI), (d->Cout + CBJ - 1) / CBJ);
  conv2d_kernel<<<grid, CONV_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_maxpool2(const float* x, float* y, int64_t planes, int32_t H, int32_t W, void* stream) {
  B200_REQUIRE(x && y && planes > 0 && H >= 2 && W >= 2, "bad arguments");
  const int64_t total = planes * (H / 2) * (W / 2);
  maxpool2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, y, planes, H, W);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_upsample_bilinear2(const float* x, float* y, int32_t N, int32_t C, int32_t H, int32_t W, int32_t out_c_total,
                            int32_t out_c_off, void* stream) {
  B200_REQUIRE(x && y && N > 0 && C > 0 && H > 0 && W > 0 && out_c_off >= 0 && out_c_off + C <= out_c_total, "bad arguments");
  const int64_t total = (int64_t)N * C * 4 * H * W;
  upsample_bilinear2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, y, N, C, H, W, out_c_total, out_c_off);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_gru_gate(const float* a, const float* b, const float* c, float* out, int64_t n_per_sample, int64_t samples,
                  int64_t out_sample_stride, int32_t mode, void* stream) {
  B200_REQUIRE(a && b && out && (mode == 0 || (mode == 1 && c)), "bad arguments");
  const int64_t total = n_per_sample * samples;
  gru_gate_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      a, b, c, out, n_per_sample, (int)out_sample_stride, mode, total);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_convlstm_cell(const float* gates, const float* prev_cell, float* hidden, float* cell, int32_t N, int32_t C,
                       int32_t H, int32_t W, void* stream) {
  B200_REQUIRE(gates && hidden && N > 0 && C > 0 && H > 0 && W > 0, "bad arguments");
  const int64_t plane = (int64_t)H * W, total = (int64_t)N * C * plane;
  convlstm_cell_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      gates, prev_cell, hidden, cell, C, plane, total);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_convlstm_zero_state(const float* gates, float* hidden, float* cell, int32_t N, int32_t C, int32_t H, int32_t W,
                             void* stream) {
  return b200_convlstm_cell(gates, nullptr, hidden, cell, N, C, H, W, stream);
}

int b200_convex_upsample(const float* flow, const float* mask, float* out, int32_t N, int32_t H, int32_t W, void* stream) {
  B200_REQUIRE(flow && mask && out && N > 0 && H > 0 && W > 0, "bad arguments");
  const int64_t total = (int64_t)N * H * W * 64;
  convex_upsample_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(flow, mask, out, N, H, W);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
