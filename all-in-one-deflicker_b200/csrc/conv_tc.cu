// wgmma implicit-GEMM convolution (fp16 operands, fp32 accumulation in registers).
//
// Same operator as conv_simt.cu (B200ConvDesc: NCHW fp32 tensors, channel slices, zero / reflection padding,
// stride, nearest x2 upsampling, bias, activation, scale, residual) for the layers whose precision in the
// reference is half / TF32 anyway: the RAFT update block runs under fp16 autocast
// (src/models/stage_1/core/raft.py:131, raft_wrapper.py:19) and the stage-2 networks run cuDNN convolutions
// with TF32 allowed (torch default) — both 10-bit-mantissa operand formats, like fp16.
//
// GEMM view: M = 128 output pixels per tile, N = output channels (tile of 64/128), K = Cin*KH*KW in chunks
// of 64.  Persistent CTAs; warp roles:
//   warps 0-7   two consumer warpgroups (64 tile rows each): wgmma (SS mode) into register accumulators, then the
//               epilogue: bias + activation + scale + residual, NCHW stores
//   warp 8      weight producer: cp.async.bulk of pre-built K-major SW128 weight images (b200_conv_weight_images)
//   warps 9-16  im2col gather, two groups of 4 warps taking alternate k chunks: each thread owns one pixel row
//               of the A tile, loads 64 taps (coalesced across the warp: consecutive pixels) through a per-CTA
//               tap table {input offset, tap id} and a per-pixel 64-bit tap-validity mask (zero padding costs
//               no branches), converts to fp16 and writes its 128-byte swizzled row
#include "common.cuh"
#include "tc_ptx.cuh"

namespace b200 {
using namespace ptx;

constexpr int CT_M = 128;
constexpr int CT_KC = 64;                       // k chunk
constexpr int CT_A_STAGES = 4, CT_B_STAGES = 3;
constexpr int CT_A_BYTES = CT_M * 128;          // 16 KB
constexpr int CT_B_BYTES = 128 * 128;           // 16 KB (N tile <= 128 rows)
constexpr int CT_CONSUMER_WARPS = 8;            // two warpgroups: wgmma + epilogue, 64 tile rows each
constexpr int CT_PRODUCER_WARP = 8;
constexpr int CT_THREADS = 544;                 // 17 warps: 8 consumer, producer, 8 gather
constexpr int CT_MAX_K = 6144;                  // padded reduction length the tap table can hold
constexpr int CT_FIXED_SMEM = CT_A_STAGES * CT_A_BYTES + CT_B_STAGES * CT_B_BYTES + 512;

struct ConvTcArgs {
  B200ConvDesc d;
  const float* x; const char* w_img; const float* bias; const float* res; float* y;
  int OH, OW, R, n_chunks;      // output size, reduction length, ceil(R / 64)
  int n_tile, n_tiles_n;        // N tile (64/128) and number of cout tiles
  int64_t pixels; int m_tiles;
};

__device__ __forceinline__ float ct_act(float v, int act) {
  switch (act) {
    case 1: return fmaxf(v, 0.f);
    case 2: return v > 0.f ? v : 0.2f * v;
    case 3: return 1.0f / (1.0f + expf(-v));
    case 4: return tanhf(v);
    default: return v;
  }
}
__device__ __forceinline__ int ct_reflect(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}
__device__ __forceinline__ int ct_atom_off(int m, int k) {
  const int r = m & 7;
  return (m >> 3) * 1024 + r * 128 + (((k >> 3) ^ r) << 4) + ((k & 7) << 1);
}

// MMAs + epilogue of the consumer warpgroups for one N-tile width
template <int NT>
__device__ __forceinline__ void ct_consume(const ConvTcArgs& a, char* sA, char* sB, uint64_t* a_full, uint64_t* a_empty,
                                           uint64_t* b_full, uint64_t* b_empty) {
  const B200ConvDesc& d = a.d;
  const int warp = warp_uniform(), lane = threadIdx.x & 31, g = warp >> 2, q = lane & 3;
  const int m0 = 64 * g + 16 * (warp & 3) + (lane >> 2);
  const int total_tiles = a.m_tiles * a.n_tiles_n;
  const int64_t oplane = (int64_t)a.OH * a.OW;
  float acc[NT / 2];
  uint32_t it = 0;
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    int pend_a = -1, pend_b = -1;
    for (int c = 0; c < a.n_chunks; ++c, ++it) {
      const int sa = it % CT_A_STAGES, sb = it % CT_B_STAGES;
      mbar_wait(&a_full[sa], (it / CT_A_STAGES) & 1);
      mbar_wait(&b_full[sb], (it / CT_B_STAGES) & 1);
      const uint32_t pa = smem_u32(sA + sa * CT_A_BYTES) + g * 8192, pb = smem_u32(sB + sb * CT_B_BYTES);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t da = make_desc(pa + ks * 32, 16, 1024), db = make_desc(pb + ks * 32, 16, 1024);
        if constexpr (NT == 128) wgmma_n128<0, 0>(acc, da, db, (c | ks) ? 1u : 0u);
        else wgmma_n64<0, 0>(acc, da, db, (c | ks) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (pend_a >= 0 && lane == 0) { mbar_arrive(&a_empty[pend_a]); mbar_arrive(&b_empty[pend_b]); }
      pend_a = sa; pend_b = sb;
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (pend_a >= 0 && lane == 0) { mbar_arrive(&a_empty[pend_a]); mbar_arrive(&b_empty[pend_b]); }
    const int mt = t / a.n_tiles_n, nt = t % a.n_tiles_n;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int64_t p = (int64_t)mt * CT_M + m0 + 8 * rr;
      if (p >= a.pixels) continue;
      const int64_t n = p / oplane, sp = p % oplane;
#pragma unroll
      for (int i = 0; i < NT / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = nt * NT + 8 * i + 2 * q + e;
          if (j < d.Cout) {
            float val = acc[4 * i + 2 * rr + e];
            if (a.bias) val += __ldg(a.bias + j);
            val = ct_act(val, d.act) * d.out_scale;
            if (a.res) val += __ldg(a.res + (n * d.res_c_total + d.res_c_off + j) * oplane + sp);
            a.y[(n * d.out_c_total + d.out_c_off + j) * oplane + sp] = val;
          }
        }
    }
  }
}

__global__ void __launch_bounds__(CT_THREADS, 1) conv2d_tc_kernel(const __grid_constant__ ConvTcArgs a) {
  extern __shared__ __align__(1024) char smem[];
  char* sA = smem;
  char* sB = smem + CT_A_STAGES * CT_A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + CT_B_STAGES * CT_B_BYTES);
  int2* ktab = reinterpret_cast<int2*>(sB + CT_B_STAGES * CT_B_BYTES + 512);     // [n_chunks * 64] {offset, tap}
  uint64_t* a_full = bars;                         // [4] 128 gather arrivals
  uint64_t* a_empty = a_full + CT_A_STAGES;        // [4] one arrival per consumer warp
  uint64_t* b_full = a_empty + CT_A_STAGES;        // [3] tx
  uint64_t* b_empty = b_full + CT_B_STAGES;        // [3] one arrival per consumer warp
  const int warp = warp_uniform(), lane = threadIdx.x & 31;
  const B200ConvDesc& d = a.d;
  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();   // the swizzled operand layouts need 1024-byte alignment
    for (int i = 0; i < CT_A_STAGES; ++i) { mbar_init(&a_full[i], 128); mbar_init(&a_empty[i], CT_CONSUMER_WARPS); }
    for (int i = 0; i < CT_B_STAGES; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], CT_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  {
    const int KHW = d.KH * d.KW, plane = d.H * d.W;
    for (int k = threadIdx.x; k < a.n_chunks * CT_KC; k += CT_THREADS) {
      const int ci = k / KHW, kk = k % KHW;
      ktab[k] = k < a.R ? make_int2(ci * plane + (kk / d.KW) * d.W + (kk % d.KW), kk) : make_int2(0, 63);
    }
  }
  __syncthreads();
  const int total_tiles = a.m_tiles * a.n_tiles_n;
  const int b_bytes = a.n_tile * 128;

  if (warp < CT_CONSUMER_WARPS) {
    if (a.n_tile == 128) ct_consume<128>(a, sA, sB, a_full, a_empty, b_full, b_empty);
    else ct_consume<64>(a, sA, sB, a_full, a_empty, b_full, b_empty);
  } else if (warp == CT_PRODUCER_WARP) {
    if (lane == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int nt = t % a.n_tiles_n;
        const char* src = a.w_img + (int64_t)nt * a.n_chunks * b_bytes;
        for (int c = 0; c < a.n_chunks; ++c, ++it) {
          const int s = it % CT_B_STAGES;
          mbar_wait(&b_empty[s], ((it / CT_B_STAGES) & 1) ^ 1);
          mbar_expect_tx(&b_full[s], b_bytes);
          bulk_g2s(sB + s * CT_B_BYTES, src + (int64_t)c * b_bytes, b_bytes, &b_full[s]);
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ im2col gather
    const int gw = warp - CT_PRODUCER_WARP - 1;             // 0..7
    const int grp = gw >> 2;                               // chunk parity this group fills
    const int m = (gw & 3) * 32 + lane;                    // row of the A tile
    const int HU = d.H * d.upsample, WU = d.W * d.upsample;
    const int KHW = d.KH * d.KW;
    const int plane = d.H * d.W;
    const uint64_t full_mask = (KHW >= 64) ? ~0ull : ((1ull << KHW) - 1);
    uint32_t it = 0;
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      const int mt = t / a.n_tiles_n;
      const int64_t p = (int64_t)mt * CT_M + m;
      const bool live = p < a.pixels;
      int py = 0, px = 0, base = 0;
      uint64_t mask = 0;
      if (live) {
        const int ox = (int)(p % a.OW), oy = (int)((p / a.OW) % a.OH);
        const int n = (int)(p / ((int64_t)a.OW * a.OH));
        py = oy * d.stride - d.pad_h; px = ox * d.stride - d.pad_w;
        base = (n * d.in_c_total + d.in_c_off) * plane;
        for (int ky = 0; ky < d.KH; ++ky)
          for (int kx = 0; kx < d.KW; ++kx)
            if (py + ky >= 0 && py + ky < HU && px + kx >= 0 && px + kx < WU) mask |= 1ull << (ky * d.KW + kx);
      }
      // branch-free path: zero padding (mask decides), or reflection padding away from the border
      const bool fast = d.upsample == 1 && (d.pad_mode == 0 || mask == full_mask || !live);
      const float* __restrict__ pp = a.x + (base + py * d.W + px);
      // every lane live, all taps in range and the table holds no padding taps in this chunk -> checked per chunk
      const bool warp_inside = __all_sync(0xffffffffu, live && mask == full_mask);
      for (int c = 0; c < a.n_chunks; ++c, ++it) {
        if ((int)(it & 1) != grp) continue;
        const int s = it % CT_A_STAGES;
        mbar_wait(&a_empty[s], ((it / CT_A_STAGES) & 1) ^ 1);
        char* row = sA + s * CT_A_BYTES;
        const int4* tab = reinterpret_cast<const int4*>(ktab + c * CT_KC);
        const bool interior = warp_inside && (c + 1) * CT_KC <= a.R;
        if (fast) {
          float v[64];
          if (interior) {                                  // whole warp away from the border: no tap test
#pragma unroll
            for (int q = 0; q < 32; ++q) {
              const int4 e = tab[q];                       // two taps: {off, tap, off, tap}
              v[2 * q] = __ldg(pp + e.x);
              v[2 * q + 1] = __ldg(pp + e.z);
            }
          } else {
#pragma unroll
            for (int q = 0; q < 32; ++q) {
              const int4 e = tab[q];
              v[2 * q] = ((mask >> e.y) & 1) ? __ldg(pp + e.x) : 0.f;
              v[2 * q + 1] = ((mask >> e.w) & 1) ? __ldg(pp + e.z) : 0.f;
            }
          }
#pragma unroll
          for (int c8 = 0; c8 < 8; ++c8) {
            const uint4 pk = make_uint4(cvt_pack_f16x2(v[c8 * 8 + 0], v[c8 * 8 + 1]), cvt_pack_f16x2(v[c8 * 8 + 2], v[c8 * 8 + 3]),
                                        cvt_pack_f16x2(v[c8 * 8 + 4], v[c8 * 8 + 5]), cvt_pack_f16x2(v[c8 * 8 + 6], v[c8 * 8 + 7]));
            *reinterpret_cast<uint4*>(row + ct_atom_off(m, c8 * 8)) = pk;
          }
        } else {
#pragma unroll 1
          for (int c8 = 0; c8 < 8; ++c8) {
            float v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const int2 e = ktab[c * CT_KC + c8 * 8 + q];
              float val = 0.f;
              if (live && e.y < 63) {
                const int ky = e.y / d.KW, kx = e.y % d.KW;
                const int cplane = e.x - ky * d.W - kx;     // ci * plane
                int iy = py + ky, ix = px + kx;
                bool ok = true;
                if (d.pad_mode == 1) { iy = ct_reflect(iy, HU); ix = ct_reflect(ix, WU); }
                else ok = (iy >= 0 && iy < HU && ix >= 0 && ix < WU);
                if (d.upsample > 1) { iy >>= 1; ix >>= 1; }
                if (ok) val = __ldg(a.x + (base + cplane + iy * d.W + ix));
              }
              v[q] = val;
            }
            const uint4 pk = make_uint4(cvt_pack_f16x2(v[0], v[1]), cvt_pack_f16x2(v[2], v[3]),
                                        cvt_pack_f16x2(v[4], v[5]), cvt_pack_f16x2(v[6], v[7]));
            *reinterpret_cast<uint4*>(row + ct_atom_off(m, c8 * 8)) = pk;
          }
        }
        fence_proxy_async_smem();
        mbar_arrive(&a_full[s]);
      }
    }
  }
}

// weights [Cout][R] fp32 -> images [n_tile_idx][chunk][n_tile rows x 64 k] fp16, K-major SW128, zero padded
__global__ void conv_weight_images_kernel(const float* __restrict__ w, char* __restrict__ img, int Cout, int R,
                                          int n_tile, int n_chunks) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // one 16-byte chunk each
  const int rows_total = ((Cout + n_tile - 1) / n_tile) * n_tile;
  if (e >= (int64_t)rows_total * n_chunks * 8) return;
  const int c8 = (int)(e % 8), chunk = (int)((e / 8) % n_chunks), row = (int)(e / (8 * n_chunks));
  const int nt = row / n_tile, lrow = row % n_tile;
  float v[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int k = chunk * 64 + c8 * 8 + q;
    v[q] = (row < Cout && k < R) ? w[(int64_t)row * R + k] : 0.f;
  }
  const uint4 pk = make_uint4(cvt_pack_f16x2(v[0], v[1]), cvt_pack_f16x2(v[2], v[3]), cvt_pack_f16x2(v[4], v[5]),
                              cvt_pack_f16x2(v[6], v[7]));
  char* dst = img + ((int64_t)nt * n_chunks + chunk) * n_tile * 128 + ct_atom_off(lrow, c8 * 8);
  *reinterpret_cast<uint4*>(dst) = pk;
}

static int pick_n_tile(int cout) { return cout > 64 ? 128 : 64; }

}  // namespace b200

using namespace b200;

extern "C" {

int64_t b200_conv_weight_image_bytes(const B200ConvDesc* d) {
  if (!d || d->Cout <= 0 || d->Cin <= 0 || d->KH <= 0 || d->KW <= 0) return -1;
  const int R = d->Cin * d->KH * d->KW, n_tile = pick_n_tile(d->Cout);
  const int64_t chunks = (R + CT_KC - 1) / CT_KC, tiles = (d->Cout + n_tile - 1) / n_tile;
  return tiles * chunks * n_tile * 128;
}

int b200_conv_weight_images(const B200ConvDesc* d, const float* w, void* images, void* stream) {
  B200_REQUIRE(d && w && images, "null pointer");
  const int R = d->Cin * d->KH * d->KW, n_tile = pick_n_tile(d->Cout), chunks = (R + CT_KC - 1) / CT_KC;
  const int rows_total = ((d->Cout + n_tile - 1) / n_tile) * n_tile;
  const int64_t total = (int64_t)rows_total * chunks * 8;
  conv_weight_images_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, reinterpret_cast<char*>(images), d->Cout, R, n_tile, chunks);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int b200_conv2d_tc(const B200ConvDesc* d, const float* x, const void* w_images, const float* bias,
                   const float* residual, float* y, void* stream) {
  B200_REQUIRE(d && d->upsample_mode == 0, "bilinear upsampling is fused only by b200_conv2d_tma");
  B200_REQUIRE(d && x && w_images && y, "null pointer");
  B200_REQUIRE(d->N > 0 && d->Cin > 0 && d->H > 0 && d->W > 0 && d->Cout > 0 && d->KH > 0 && d->KW > 0 && d->stride > 0 &&
               (d->upsample == 1 || d->upsample == 2) && (d->pad_mode == 0 || d->pad_mode == 1) && d->act >= 0 && d->act <= 4,
               "invalid convolution descriptor");
  B200_REQUIRE(d->in_c_off >= 0 && d->in_c_off + d->Cin <= d->in_c_total && d->out_c_off >= 0 &&
               d->out_c_off + d->Cout <= d->out_c_total, "channel slice out of range");
  if (!b200_device_supports_tc()) { set_error("b200_conv2d_tc needs a compute-capability 9.x device"); return B200_ERR_UNSUPPORTED; }
  static bool attr_done = false;
  if (!attr_done) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(conv2d_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         CT_FIXED_SMEM + CT_MAX_K * 8));
    attr_done = true;
  }
  ConvTcArgs a{};
  a.d = *d; a.x = x; a.w_img = reinterpret_cast<const char*>(w_images); a.bias = bias; a.res = residual; a.y = y;
  const int HU = d->H * d->upsample, WU = d->W * d->upsample;
  B200_REQUIRE(d->pad_mode == 0 || (d->pad_h < HU && d->pad_w < WU), "reflection padding larger than the input");
  a.OH = (HU + 2 * d->pad_h - d->KH) / d->stride + 1;
  a.OW = (WU + 2 * d->pad_w - d->KW) / d->stride + 1;
  B200_REQUIRE(a.OH > 0 && a.OW > 0, "empty output");
  a.R = d->Cin * d->KH * d->KW;
  a.n_chunks = (a.R + CT_KC - 1) / CT_KC;
  B200_REQUIRE(a.n_chunks * CT_KC <= CT_MAX_K && d->KH * d->KW < 63, "reduction too long for b200_conv2d_tc (Cin*KH*KW <= 6144)");
  B200_REQUIRE((int64_t)d->N * d->in_c_total * d->H * d->W < (1ll << 31), "input too large for 32-bit offsets");
  a.n_tile = pick_n_tile(d->Cout);
  a.n_tiles_n = (d->Cout + a.n_tile - 1) / a.n_tile;
  a.pixels = (int64_t)d->N * a.OH * a.OW;
  a.m_tiles = (int)((a.pixels + CT_M - 1) / CT_M);
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t tiles = (int64_t)a.m_tiles * a.n_tiles_n;
  conv2d_tc_kernel<<<(unsigned)(tiles < sms ? tiles : sms), CT_THREADS, CT_FIXED_SMEM + a.n_chunks * CT_KC * 8, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // extern "C"
