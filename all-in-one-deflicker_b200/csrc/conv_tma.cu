// TMA-fed wgmma convolution (fp16 operands, fp32 accumulation in registers) — no im2col gather at all.
//
// With a channels-last fp16 copy of the input, the A operand of the implicit GEMM for ONE filter tap (ky,kx)
// and one block of 64 input channels is a plain 2-D box of the tensor: 128 consecutive output pixels of one
// image row x 64 channels.  A tiled TMA load with the 128-byte swizzle lands it in shared memory in exactly the
// canonical K-major layout wgmma reads; the tap only shifts the box coordinates (the pixel dimension is
// not the innermost one, so any shift is legal for the TMA unit).  The reduction runs over (tap, channel block).
//
// Two kernels per convolution:
//   conv_pack_input_kernel  fp32 NCHW (channel slice) -> fp16 NHWC (channels padded to 64) through a shared-
//                           memory transpose, with the padding (zeros / reflection), the nearest x2 upsampling
//                           and — for stride 2 — a split into the 4 pixel phases materialised, so that the
//                           convolution proper is a stride-1 "valid" one (HBM-bound)
//   conv2d_tma_kernel       persistent, warps 0-7 = two consumer warpgroups (wgmma on 64 pixels each, then the
//                           epilogue: bias, activation, scale, residual, NCHW fp32 / packed fp16 stores),
//                           warp 8 = TMA producer (1 activation box + 1 weight image per stage)
// and convlstm_tma_kernel, the same pipeline for a ConvLSTM gate convolution whose epilogue applies the cell update
// (gate-interleaved weight image, see LstmArgs) instead of storing the gates.
//
// Same operator semantics as b200_conv2d (reference: nn.Conv2d / ReflectionPad2d / nn.Upsample call sites in
// src/models/stage_1/core/update.py, src/models/network_filter.py, src/models/network_local.py).
#include <cuda.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace b200 {
using namespace ptx;

constexpr int TM_THREADS = 384;                 // 2 consumer warpgroups + the producer warpgroup (one active lane)
constexpr int TM_CONSUMER_WARPS = 8;
constexpr int TM_MAX_A = 8, TM_MAX_B = 16;
constexpr int TM_BAR_BYTES = 1024;              // mbarriers
constexpr int TM_SMEM_BUDGET = 225 * 1024;             // of the 227 KB a block may use

struct ConvTmaArgs {
  B200ConvDesc d;
  const char* w_img; const float* bias; const float* res; float* y;
  int OH, OW, x_tiles, cchunks, n_chunks, n_tile, n_tiles_n, phases, shift, total_tiles;
  int a_rows, a_stage, n_a, n_b;                       // box rows, bytes per A stage, ring depths
  int b_group, b_stage;                                // weight chunks (x taps) per B stage, bytes per B stage
  int split;                                           // 1: both operands are (hi, lo) fp16 pairs, 3 MMAs per product
  int resident;                                        // 1: the whole weight image stays in shared memory (narrow layers)
  // chained output: the result is ALSO (or only, y == nullptr) written as fp16 into the packed input of the next
  // convolution: [n][yp_hp2][yp_wp2][yp_cp] with its zero halo (yp_pad_h, yp_pad_w), at channel offset yp_c_off
  __half* yp; int yp_hp2, yp_wp2, yp_cp, yp_pad_h, yp_pad_w, yp_c_off;
};

// ConvLSTM epilogue (convlstm_tma_kernel): the gate convolution's Cout = 4C columns come from a gate-interleaved weight
// image (column 32b + 8k + r of an N tile = gate k of hidden channel 8b + r of that tile, gates in chunk(4, 1) order:
// in, remember, out, cell), so every thread holds the four gates of its hidden channels.  NCHW fp32 [N][C][OH][OW].
struct LstmArgs {
  const float* prev_cell;                              // nullptr: zero state
  float* hidden; float* cell;                          // cell may be nullptr
  int C;
};

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}

template <int ACT>
__device__ __forceinline__ float tm_act(float v) {
  if (ACT == 1) return fmaxf(v, 0.f);
  if (ACT == 2) return v > 0.f ? v : 0.2f * v;
  if (ACT == 3) return 1.0f / (1.0f + expf(-v));
  if (ACT == 4) return tanhf(v);
  return v;
}

__device__ __forceinline__ float tm_sigmoid(float v) { return 1.0f / (1.0f + expf(-v)); }

// Consumer warpgroups for one N-tile width: the MMAs of a tile (this warpgroup's 64 pixels), then the epilogue on the
// accumulator registers (bias, activation, scale, residual; NCHW fp32 stores and / or the fp16 channel pairs of the
// next layer's packed input), or with LSTM the ConvLSTM cell update (hidden / cell stores; the gates are never stored)
template <int NT, int ACT, bool LSTM>
__device__ __forceinline__ void tma_consume(const ConvTmaArgs& a, const LstmArgs& l, char* sA, char* sB, uint64_t* a_full,
                                            uint64_t* a_empty, uint64_t* b_full, uint64_t* b_empty) {
  const B200ConvDesc& d = a.d;
  const int warp = warp_uniform(), lane = threadIdx.x & 31, g = warp >> 2, q = lane & 3;
  const int m0 = 64 * g + 16 * (warp & 3) + (lane >> 2);
  const int b_half = a.n_tile * 128;
  const int b_bytes = a.split ? 2 * b_half : b_half;
  const int a_half = a.a_stage >> 1;
  const int s = d.stride;
  const int64_t oplane = (int64_t)a.OH * a.OW;
  int sa = 0, sb = 0;
  uint32_t pha = 0, phb = 0;
  if (a.resident) mbar_wait(&b_full[0], 0);
  float acc[NT / 2];
  for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
    uint32_t accum = 0;
    int jres = 0;                                          // resident mode: index of the next weight chunk
    for (int ky = 0; ky < d.KH; ++ky)
      for (int xpar = 0; xpar < s && xpar < d.KW; ++xpar) {
        const int nsub = (d.KW - xpar + s - 1) / s;
        for (int cc = 0; cc < a.cchunks; ++cc) {
          mbar_wait(&a_full[sa], pha);
          const uint32_t pa = smem_u32(sA + sa * a.a_stage) + g * 8192;
          const int left = d.Cin - cc * 64;
          const int ksteps = ((left < 64 ? left : 64) + 15) >> 4;
          for (int i0 = 0; i0 < nsub; i0 += (a.resident ? nsub : a.b_group)) {
            const int gn = a.resident ? nsub : (nsub - i0 < a.b_group ? nsub - i0 : a.b_group);
            uint32_t pb;
            if (a.resident) {
              pb = smem_u32(sB) + jres * b_bytes;
              jres += nsub;
            } else {
              mbar_wait(&b_full[sb], phb);
              pb = smem_u32(sB + sb * a.b_stage);
            }
            wgmma_fence();
            for (int i = 0; i < gn; ++i) {
              const uint32_t ai = pa + (i0 + i) * 128, bi = pb + i * b_bytes;
              for (int ks = 0; ks < ksteps; ++ks, accum = 1u) {
                const uint64_t da = make_desc(ai + ks * 32, 16, 1024), db = make_desc(bi + ks * 32, 16, 1024);
                if constexpr (NT == 256) wgmma_n256<0, 0>(acc, da, db, accum);
                else if constexpr (NT == 128) wgmma_n128<0, 0>(acc, da, db, accum);
                else wgmma_n64<0, 0>(acc, da, db, accum);
                if (a.split) {                             // (hi + lo)(hi + lo) without the lo*lo term
                  const uint64_t da_lo = make_desc(ai + a_half + ks * 32, 16, 1024);
                  const uint64_t db_lo = make_desc(bi + b_half + ks * 32, 16, 1024);
                  if constexpr (NT == 256) { wgmma_n256<0, 0>(acc, da, db_lo, 1u); wgmma_n256<0, 0>(acc, da_lo, db, 1u); }
                  else if constexpr (NT == 128) { wgmma_n128<0, 0>(acc, da, db_lo, 1u); wgmma_n128<0, 0>(acc, da_lo, db, 1u); }
                  else { wgmma_n64<0, 0>(acc, da, db_lo, 1u); wgmma_n64<0, 0>(acc, da_lo, db, 1u); }
                }
              }
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (!a.resident) {
              if (lane == 0) mbar_arrive(&b_empty[sb]);
              if (++sb == a.n_b) { sb = 0; phb ^= 1; }
            }
          }
          if (lane == 0) mbar_arrive(&a_empty[sa]);
          if (++sa == a.n_a) { sa = 0; pha ^= 1; }
        }
      }
    acc_fence(acc);
    const int nt = t % a.n_tiles_n;
    int r = t / a.n_tiles_n;
    const int xb = r % a.x_tiles; r /= a.x_tiles;
    const int oy = r % a.OH, n = r / a.OH;
    if constexpr (LSTM) {
      // accumulator column 8i + 2q + e with i = 4b + k: gate k of hidden channel h0 + 8b + 2q + e (C % 8 == 0, so a
      // channel pair lies inside [0, C) or outside it together)
      const int C = l.C, h0 = nt * (NT / 4);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int x = xb * 128 + m0 + 8 * rr;
        if (x >= a.OW) continue;
        const int64_t pix = (int64_t)n * C * oplane + (int64_t)oy * a.OW + x;
#pragma unroll
        for (int b = 0; b < NT / 32; ++b) {
          const int hc = h0 + 8 * b + 2 * q;
          if (hc >= C) continue;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int h = hc + e;
            float gv[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              gv[k] = acc[4 * (4 * b + k) + 2 * rr + e];
              if (a.bias) gv[k] += __ldg(a.bias + k * C + h);
            }
            // the expressions of convlstm_cell_kernel (conv_simt.cu), so both paths agree on the same gates
            const float in_g = tm_sigmoid(gv[0]), out_g = tm_sigmoid(gv[2]), cell_g = tanhf(gv[3]);
            const int64_t o = pix + (int64_t)h * oplane;
            float cl;
            if (l.prev_cell)                                // torch: (remember * prev) + (in * cell_gate), each rounded
              cl = __fadd_rn(__fmul_rn(tm_sigmoid(gv[1]), __ldg(l.prev_cell + o)), __fmul_rn(in_g, cell_g));
            else
              cl = in_g * cell_g;
            l.hidden[o] = out_g * tanhf(cl);
            if (l.cell) l.cell[o] = cl;
          }
        }
      }
      continue;
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int x = xb * 128 + m0 + 8 * rr;
      if (x >= a.OW) continue;
      const int64_t sp = (int64_t)oy * a.OW + x;
      const float* resp = a.res ? a.res + ((int64_t)n * d.res_c_total + d.res_c_off) * oplane + sp : nullptr;
      float* yp = a.y ? a.y + ((int64_t)n * d.out_c_total + d.out_c_off) * oplane + sp : nullptr;
      __half* ypix = a.yp ? a.yp + ((((int64_t)n * a.yp_hp2 + oy + a.yp_pad_h) * a.yp_wp2 + x + a.yp_pad_w) * a.yp_cp +
                                    a.yp_c_off) : nullptr;
#pragma unroll
      for (int i = 0; i < NT / 8; ++i) {
        const int j = nt * a.n_tile + 8 * i + 2 * q;
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float val = acc[4 * i + 2 * rr + e];
          if (j + e < d.Cout) {
            if (a.bias) val += __ldg(a.bias + j + e);
            val = tm_act<ACT>(val) * d.out_scale;
            if (resp) val += __ldg(resp + (int64_t)(j + e) * oplane);
            if (yp) yp[(int64_t)(j + e) * oplane] = val;
          }
          v[e] = val;
        }
        // saturating like the repack (split2_f16), so a chained consumer sees the operands an unchained one would
        if (ypix && j < d.Cout) *reinterpret_cast<uint32_t*>(ypix + j) = cvt_pack_f16x2(v[0], v[1]);   // Cout % 8 == 0 here
      }
    }
  }
}

template <int NT, bool LSTM>
__device__ __forceinline__ void tma_consume_act(const ConvTmaArgs& a, const LstmArgs& l, char* sA, char* sB,
                                                uint64_t* a_full, uint64_t* a_empty, uint64_t* b_full,
                                                uint64_t* b_empty) {
  if constexpr (LSTM) {                                  // no activation, scale or residual in front of the cell
    tma_consume<NT, 0, true>(a, l, sA, sB, a_full, a_empty, b_full, b_empty);
    return;
  }
  switch (a.d.act) {
    case 1: tma_consume<NT, 1, false>(a, l, sA, sB, a_full, a_empty, b_full, b_empty); break;
    case 2: tma_consume<NT, 2, false>(a, l, sA, sB, a_full, a_empty, b_full, b_empty); break;
    case 3: tma_consume<NT, 3, false>(a, l, sA, sB, a_full, a_empty, b_full, b_empty); break;
    case 4: tma_consume<NT, 4, false>(a, l, sA, sB, a_full, a_empty, b_full, b_empty); break;
    default: tma_consume<NT, 0, false>(a, l, sA, sB, a_full, a_empty, b_full, b_empty); break;
  }
}

// Reduction order shared by the producer, the consumers and the weight images:
//   for ky, for xpar in [0, stride), for cc (64-channel block):   one activation box (all x shifts of that row)
//     for kx = xpar, xpar + stride, ... < KW:                      one weight chunk, A start shifted by kx>>shift rows
template <bool LSTM>
__device__ __forceinline__ void conv_tma_body(const ConvTmaArgs& a, const CUtensorMap& xmap, const CUtensorMap& xmap_lo,
                                              const LstmArgs& l) {
  extern __shared__ __align__(1024) char smem[];
  const int b_half = a.n_tile * 128;                    // one term of one weight chunk
  const int b_bytes = a.split ? 2 * b_half : b_half;
  char* sA = smem;
  char* sB = smem + a.n_a * a.a_stage;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + a.n_b * a.b_stage);
  uint64_t* a_full = bars;                         // tx
  uint64_t* a_empty = a_full + TM_MAX_A;           // one arrival per consumer warp
  uint64_t* b_full = a_empty + TM_MAX_A;           // tx
  uint64_t* b_empty = b_full + TM_MAX_B;           // one arrival per consumer warp
  const int warp = warp_uniform(), lane = threadIdx.x & 31;
  const B200ConvDesc& d = a.d;
  if (threadIdx.x == 0) {
    if (smem_u32(smem) & 1023u) __trap();   // the swizzled operand layouts need 1024-byte alignment
    for (int i = 0; i < TM_MAX_A; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], TM_CONSUMER_WARPS); }
    for (int i = 0; i < TM_MAX_B; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], TM_CONSUMER_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();
  const int s = d.stride;

  if (warp < TM_CONSUMER_WARPS) {
    setmaxnreg_inc<232>();                               // 128 * 40 + 256 * 232 <= 64 K
    if (a.n_tile == 256) tma_consume_act<256, LSTM>(a, l, sA, sB, a_full, a_empty, b_full, b_empty);
    else if (a.n_tile == 128) tma_consume_act<128, LSTM>(a, l, sA, sB, a_full, a_empty, b_full, b_empty);
    else tma_consume_act<64, LSTM>(a, l, sA, sB, a_full, a_empty, b_full, b_empty);
    return;
  }
  setmaxnreg_dec<40>();
  if (warp == TM_CONSUMER_WARPS && lane == 0) {
    int sa = 0, sb = 0;
    uint32_t pha = 0, phb = 0;
    if (a.resident) {                                      // one cout tile, all chunks: loaded once per CTA
      mbar_expect_tx(&b_full[0], a.n_chunks * b_bytes);
      for (int j = 0; j < a.n_chunks; ++j) bulk_g2s(sB + j * b_bytes, a.w_img + (int64_t)j * b_bytes, b_bytes, &b_full[0]);
    }
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
      const int nt = t % a.n_tiles_n;
      int r = t / a.n_tiles_n;
      const int xb = r % a.x_tiles; r /= a.x_tiles;
      const int oy = r % a.OH, n = r / a.OH;
      const char* wsrc = a.w_img + (int64_t)nt * a.n_chunks * b_bytes;
      for (int ky = 0; ky < d.KH; ++ky)
        for (int xpar = 0; xpar < s && xpar < d.KW; ++xpar) {
          const int nsub = (d.KW - xpar + s - 1) / s;
          const int ph = a.phases == 4 ? ((ky & 1) * 2 + xpar) : 0;
          for (int cc = 0; cc < a.cchunks; ++cc) {
            mbar_wait(&a_empty[sa], pha ^ 1);
            mbar_expect_tx(&a_full[sa], a.a_rows * 128 * (1 + a.split));
            tma_load_4d(sA + sa * a.a_stage, &xmap, cc * 64, xb * 128, oy + (ky >> a.shift), n * a.phases + ph, &a_full[sa]);
            if (a.split)
              tma_load_4d(sA + sa * a.a_stage + (a.a_stage >> 1), &xmap_lo, cc * 64, xb * 128, oy + (ky >> a.shift),
                          n * a.phases + ph, &a_full[sa]);
            if (++sa == a.n_a) { sa = 0; pha ^= 1; }
            if (a.resident) continue;
            for (int i0 = 0; i0 < nsub; i0 += a.b_group) {
              const int gn = nsub - i0 < a.b_group ? nsub - i0 : a.b_group;
              mbar_wait(&b_empty[sb], phb ^ 1);
              mbar_expect_tx(&b_full[sb], gn * b_bytes);
              bulk_g2s(sB + sb * a.b_stage, wsrc, gn * b_bytes, &b_full[sb]);
              wsrc += gn * b_bytes;
              if (++sb == a.n_b) { sb = 0; phb ^= 1; }
            }
          }
        }
    }
  }
}

__global__ void __launch_bounds__(TM_THREADS, 1) conv2d_tma_kernel(const __grid_constant__ ConvTmaArgs a,
                                                                   const __grid_constant__ CUtensorMap xmap,
                                                                   const __grid_constant__ CUtensorMap xmap_lo) {
  conv_tma_body<false>(a, xmap, xmap_lo, LstmArgs{});
}

// the ConvLSTM gate convolution with the cell update in its epilogue (gate-interleaved weight image, see LstmArgs)
__global__ void __launch_bounds__(TM_THREADS, 1) convlstm_tma_kernel(const __grid_constant__ ConvTmaArgs a,
                                                                     const __grid_constant__ CUtensorMap xmap,
                                                                     const __grid_constant__ CUtensorMap xmap_lo,
                                                                     const __grid_constant__ LstmArgs l) {
  conv_tma_body<true>(a, xmap, xmap_lo, l);
}

__device__ __forceinline__ int tm_reflect(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// fp32 NCHW slice -> fp16 [N*phases][HP2][WP2][Cp] (Cp = channels padded to 64) with padding / upsampling /
// phase split applied.  One block = 32 pixels of one row x 64 channels, transposed through shared memory.
// Channels [0, c_write) of the slice land at channel c_off of each packed pixel (a whole repack: c_off = 0, c_write =
// Cp, the padding channels written as zeros; a slice into a shared packed input: c_write = Cin, c_off % 8 == 0).
__global__ void __launch_bounds__(256) conv_pack_input_kernel(const float* __restrict__ x, __half* __restrict__ xp,
                                                              B200ConvDesc d, int HP2, int WP2, int Cp, int phases,
                                                              float scale, int64_t lo_off, int fold_cf, int c_off,
                                                              int c_write) {
  __shared__ float tile[64][33];
  const int cblocks = (c_write + 63) / 64;
  const int cb = blockIdx.z % cblocks, nph = blockIdx.z / cblocks;
  const int ph = nph % phases, n = nph / phases;
  const int yy = blockIdx.y, bx = blockIdx.x * 32;
  const int s = d.stride, HU = d.H * d.upsample, WU = d.W * d.upsample;
  {
    const int lx_ = threadIdx.x & 31, crow = threadIdx.x >> 5;
    if (fold_cf) {
      // channel slot k = kx * fold_cf + c holds input channel c at x + kx (stride 1, nearest sampling only)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int k = crow + 8 * i, kx = k / fold_cf, c = k - kx * fold_cf;
        const int Y = yy - d.pad_h, X = bx + lx_ + kx - d.pad_w;
        int u = Y, w = X;
        bool ok = kx < d.KW && c < d.Cin && bx + lx_ < WP2;
        if (d.pad_mode == 1) { u = tm_reflect(Y, HU); w = tm_reflect(X, WU); ok = ok && Y >= -d.pad_h && Y < HU + d.pad_h; }
        else ok = ok && Y >= 0 && Y < HU && X >= 0 && X < WU;
        if (d.upsample > 1) { u >>= 1; w >>= 1; }
        tile[k][lx_] = ok ? __ldg(x + ((int64_t)n * d.in_c_total + d.in_c_off + c) * d.H * d.W + (int64_t)u * d.W + w) : 0.f;
      }
    } else {
    const int Y = yy * s + (phases == 4 ? (ph >> 1) : 0) - d.pad_h;
    const int X = (bx + lx_) * s + (phases == 4 ? (ph & 1) : 0) - d.pad_w;
    int u = Y, w = X;
    bool ok;
    if (d.pad_mode == 1) {
      ok = Y >= -d.pad_h && Y < HU + d.pad_h && X >= -d.pad_w && X < WU + d.pad_w && bx + lx_ < WP2;
      u = tm_reflect(Y, HU); w = tm_reflect(X, WU);
    } else {
      ok = Y >= 0 && Y < HU && X >= 0 && X < WU;
    }
    const int64_t plane = (int64_t)d.H * d.W;
    const float* src0 = x + ((int64_t)n * d.in_c_total + d.in_c_off) * plane;
    if (d.upsample > 1 && d.upsample_mode == 1) {
      // bilinear x2, align_corners=True (ATen area_pixel_compute_source_index): src = dst * (in-1)/(out-1)
      const float sh = HU > 1 ? (float)(d.H - 1) / (float)(HU - 1) : 0.f;
      const float sw = WU > 1 ? (float)(d.W - 1) / (float)(WU - 1) : 0.f;
      const float fy = sh * u, fx = sw * w;
      const int y0 = (int)fy, x0 = (int)fx;
      const int y1 = y0 + (y0 < d.H - 1 ? 1 : 0), x1 = x0 + (x0 < d.W - 1 ? 1 : 0);
      const float ly = fy - y0, lx = fx - x0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = cb * 64 + crow + 8 * i;
        float v = 0.f;
        if (ok && c < d.Cin) {
          const float* s = src0 + (int64_t)c * plane;
          v = (1.f - ly) * ((1.f - lx) * __ldg(s + y0 * d.W + x0) + lx * __ldg(s + y0 * d.W + x1)) +
              ly * ((1.f - lx) * __ldg(s + y1 * d.W + x0) + lx * __ldg(s + y1 * d.W + x1));
        }
        tile[crow + 8 * i][lx_] = v;
      }
    } else {
      if (d.upsample > 1) { u >>= 1; w >>= 1; }
      const float* src = src0 + (int64_t)u * d.W + w;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = cb * 64 + crow + 8 * i;
        tile[crow + 8 * i][lx_] = (ok && c < d.Cin) ? __ldg(src + (int64_t)c * plane) : 0.f;
      }
    }
    }
  }
  __syncthreads();
  const int px = threadIdx.x >> 3, c8 = threadIdx.x & 7;
  if (bx + px < WP2 && cb * 64 + c8 * 8 < c_write) {
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = tile[c8 * 8 + q][px] * scale;
    uint4 hi, lo;
    split2_f16(v[0], v[1], hi.x, lo.x); split2_f16(v[2], v[3], hi.y, lo.y);
    split2_f16(v[4], v[5], hi.z, lo.z); split2_f16(v[6], v[7], hi.w, lo.w);
    const int64_t o = (((int64_t)nph * HP2 + yy) * WP2 + bx + px) * Cp + c_off + cb * 64 + c8 * 8;
    *reinterpret_cast<uint4*>(xp + o) = hi;
    if (lo_off) *reinterpret_cast<uint4*>(xp + lo_off + o) = lo;
  }
}

// nn.ReflectionPad2d on a packed input whose interior was written by the producing convolutions: every halo pixel of
// [N][HP2][WP2][Cp] copies the vector of its mirror pixel.  One thread per (halo pixel, 8-channel group).
__global__ void conv_reflect_halo_kernel(__half* __restrict__ xp, int N, int H, int W, int pad_h, int pad_w, int Cp) {
  const int HP2 = H + 2 * pad_h, WP2 = W + 2 * pad_w;
  const int c8n = Cp / 8;
  const int64_t halo_px = (int64_t)HP2 * WP2 - (int64_t)H * W;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)N * halo_px * c8n) return;
  const int c8 = (int)(i % c8n);
  int64_t r = i / c8n;
  const int n = (int)(r / halo_px);
  r -= (int64_t)n * halo_px;
  // halo pixels in order: pad_h full rows on top, pad_h full rows at the bottom, then the side columns of the H rows
  int Y, X;
  const int64_t band = (int64_t)pad_h * WP2;
  if (r < band) { Y = (int)(r / WP2); X = (int)(r % WP2); }
  else if (r < 2 * band) { r -= band; Y = pad_h + H + (int)(r / WP2); X = (int)(r % WP2); }
  else {
    r -= 2 * band;
    Y = pad_h + (int)(r / (2 * pad_w));
    const int k = (int)(r % (2 * pad_w));
    X = k < pad_w ? k : W + k;                     // left columns 0..pad_w-1, right columns pad_w+W ..
  }
  const int sy = tm_reflect(Y - pad_h, H) + pad_h, sx = tm_reflect(X - pad_w, W) + pad_w;
  const uint4 v = *reinterpret_cast<const uint4*>(xp + (((int64_t)n * HP2 + sy) * WP2 + sx) * Cp + c8 * 8);
  *reinterpret_cast<uint4*>(xp + (((int64_t)n * HP2 + Y) * WP2 + X) * Cp + c8 * 8) = v;
}

// weights [Cout][Cin][KH][KW] fp32 -> per cout tile, per (tap, channel block): [n_tile rows x 64 channels] fp16,
// K-major, 128-byte swizzle, zero padded
// (w_co, w_ci, w_tap = element strides of the weight tensor; split: chunk = [hi rows | lo rows], values pre-scaled;
// lstm_c > 0: gate-interleaved rows for convlstm_tma_kernel, Cout = 4 * lstm_c: row 32b + 8k + r of cout tile nt holds
// weight row k * lstm_c + nt * n_tile / 4 + 8b + r, i.e. gate k of that hidden channel)
__global__ void conv_tma_weight_images_kernel(const float* __restrict__ w, char* __restrict__ img, int Cout, int Cin,
                                              int KH, int KW, int stride, int n_tile, int n_tiles_n, int cchunks,
                                              int64_t w_co, int64_t w_ci, int64_t w_tap, float scale, int split,
                                              int fold_cf, int lstm_c) {
  const int KHW = KH * KW, n_chunks = fold_cf ? KH : KHW * cchunks;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // one 16-byte chunk each
  if (e >= (int64_t)n_tiles_n * n_tile * n_chunks * 8) return;
  const int c8 = (int)(e % 8), j = (int)((e / 8) % n_chunks), grow = (int)(e / (8 * n_chunks));
  const int nt = grow / n_tile, lrow = grow % n_tile;
  int row = nt * n_tile + lrow;
  if (lstm_c) {
    const int hc = nt * (n_tile >> 2) + (lrow >> 5) * 8 + (lrow & 7);
    row = hc < lstm_c ? ((lrow >> 3) & 3) * lstm_c + hc : Cout;        // Cout: a zero row
  }
  // chunk j -> (ky, xpar, cc, kx) in the kernel's reduction order
  int tap = 0, cc = 0;
  if (!fold_cf) {
    int cnt = 0;
    bool found = false;
    for (int ky = 0; ky < KH && !found; ++ky)
      for (int xpar = 0; xpar < stride && xpar < KW && !found; ++xpar)
        for (int c = 0; c < cchunks && !found; ++c)
          for (int kx = xpar; kx < KW; kx += stride, ++cnt)
            if (cnt == j) { tap = ky * KW + kx; cc = c; found = true; break; }
  }
  float v[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    int ci = cc * 64 + c8 * 8 + q, tp = tap;
    bool ok = row < Cout;
    if (fold_cf) {                                         // chunk j = filter row, slot k = kx * fold_cf + c
      const int kx = ci / fold_cf;
      ci -= kx * fold_cf; tp = j * KW + kx; ok = ok && kx < KW;
    }
    v[q] = (ok && ci < Cin) ? w[row * w_co + ci * w_ci + tp * w_tap] * scale : 0.f;
  }
  uint4 hi, lo;
  split2_f16(v[0], v[1], hi.x, lo.x); split2_f16(v[2], v[3], hi.y, lo.y);
  split2_f16(v[4], v[5], hi.z, lo.z); split2_f16(v[6], v[7], hi.w, lo.w);
  const int rr = lrow & 7;
  const int64_t chunk_bytes = (int64_t)n_tile * 128 * (1 + split);
  char* dst = img + ((int64_t)nt * n_chunks + j) * chunk_bytes + (lrow >> 3) * 1024 + rr * 128 + ((c8 ^ rr) << 4);
  *reinterpret_cast<uint4*>(dst) = hi;
  if (split) *reinterpret_cast<uint4*>(dst + (int64_t)n_tile * 128) = lo;
}

struct TmaGeom {
  int HU, WU, OH, OW, phases, shift, HP2, WP2, Cp, cchunks, n_chunks, n_tile, n_tiles_n;
  int a_rows;       // pixel rows of one activation box: 128 outputs plus the x taps that share it
  int fold_cf;      // > 0: the KW x taps are folded into the channel dimension, fold_cf channels per tap (narrow inputs)
  int64_t pack_bytes;
};

static int tma_geometry(const B200ConvDesc* d, TmaGeom* g) {
  B200_REQUIRE(d, "null descriptor");
  B200_REQUIRE(d->N > 0 && d->Cin > 0 && d->H > 0 && d->W > 0 && d->Cout > 0 && d->KH > 0 && d->KW > 0 &&
               (d->stride == 1 || d->stride == 2) && (d->upsample == 1 || d->upsample == 2) &&
               (d->pad_mode == 0 || d->pad_mode == 1) && d->act >= 0 && d->act <= 4 && d->pad_h >= 0 && d->pad_w >= 0 &&
               (d->upsample_mode == 0 || (d->upsample_mode == 1 && d->upsample == 2)),
               "invalid convolution descriptor (b200_conv2d_tma_chain supports stride 1 and 2)");
  g->HU = d->H * d->upsample; g->WU = d->W * d->upsample;
  B200_REQUIRE(d->pad_mode == 0 || (d->pad_h < g->HU && d->pad_w < g->WU), "reflection padding larger than the input");
  const int HP = g->HU + 2 * d->pad_h, WP = g->WU + 2 * d->pad_w;
  B200_REQUIRE(HP >= d->KH && WP >= d->KW, "empty output");
  g->OH = (HP - d->KH) / d->stride + 1; g->OW = (WP - d->KW) / d->stride + 1;
  g->phases = d->stride == 2 ? 4 : 1; g->shift = d->stride == 2 ? 1 : 0;
  g->HP2 = (HP + d->stride - 1) / d->stride;
  g->WP2 = (WP + d->stride - 1) / d->stride;
  g->cchunks = (d->Cin + 63) / 64;
  g->n_chunks = d->KH * d->KW * g->cchunks;
  g->Cp = g->cchunks * 64;
  // narrow inputs (Cin <= 8 for 7-wide filters, <= 16 for 3-wide ...): pack the KW horizontally shifted copies of a
  // pixel next to each other in its 64-channel vector; the convolution then has KW = 1 and one chunk per filter row
  g->fold_cf = 0;
  const int cf = (d->Cin + 7) / 8 * 8;
  if (d->stride == 1 && d->KW > 1 && cf * d->KW <= 64 && d->upsample_mode == 0) {
    g->fold_cf = cf;
    g->WP2 = g->OW;
    g->n_chunks = d->KH;
  }
  g->a_rows = 128 + (((g->fold_cf ? 1 : d->KW) - 1) >> g->shift);   // folded: the x taps live in the channel dimension
  B200_REQUIRE(g->a_rows <= 256, "filter too wide");                // the TMA box holds at most 256 rows
  g->n_tiles_n = (d->Cout + 255) / 256;
  const int per_tile = (d->Cout + g->n_tiles_n - 1) / g->n_tiles_n;
  g->n_tile = per_tile <= 64 ? 64 : (per_tile <= 128 ? 128 : 256);   // the wgmma N shapes the kernel is built for
  g->pack_bytes = (int64_t)d->N * g->phases * g->HP2 * g->WP2 * g->Cp * 2;
  return B200_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int launch_weight_images(const B200ConvDesc* d, const TmaGeom& g, const float* w, int64_t w_co, int64_t w_ci,
                                int64_t w_tap, float scale, int split, void* images, cudaStream_t st, int lstm_c = 0) {
  const int64_t total = (int64_t)g.n_tiles_n * g.n_tile * g.n_chunks * 8;
  conv_tma_weight_images_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
      w, reinterpret_cast<char*>(images), d->Cout, d->Cin, d->KH, d->KW, d->stride, g.n_tile, g.n_tiles_n, g.cchunks, w_co,
      w_ci, w_tap, scale, split, g.fold_cf, lstm_c);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// repack x into `base` (fp16, hi then lo when split) and run the convolution
struct ChainOut { __half* yp = nullptr; int hp2 = 0, wp2 = 0, cp = 0, pad_h = 0, pad_w = 0, c_off = 0; };

// x == nullptr: `base` already holds the packed input (written by the producing convolution's epilogue)
// lstm != nullptr: the ConvLSTM gate layer (convlstm_tma_kernel; y, residual and chain unused)
static int launch_conv_tma(const B200ConvDesc* d, const TmaGeom& g, const float* x, char* base, const void* w_images,
                           const float* bias, const float* residual, float* y, int split, float in_scale, cudaStream_t st,
                           const ChainOut* chain = nullptr, const LstmArgs* lstm = nullptr) {
  B200_REQUIRE(g.HP2 <= 65535 && (int64_t)d->N * g.phases * g.cchunks <= 65535, "input too large for the repack grid");
  if (x) {
    conv_pack_input_kernel<<<dim3((g.WP2 + 31) / 32, g.HP2, d->N * g.phases * g.cchunks), 256, 0, st>>>(
        x, reinterpret_cast<__half*>(base), *d, g.HP2, g.WP2, g.Cp, g.phases, in_scale, split ? g.pack_bytes / 2 : 0, g.fold_cf,
        0, g.Cp);
    B200_CHECK_LAUNCH();
  }

  EncodeTiledFn enc = encode_tiled();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return B200_ERR_UNSUPPORTED; }
  alignas(64) CUtensorMap map, map_lo;
  const cuuint64_t dims[4] = {(cuuint64_t)g.Cp, (cuuint64_t)g.WP2, (cuuint64_t)g.HP2, (cuuint64_t)d->N * g.phases};
  const cuuint64_t strides[3] = {(cuuint64_t)g.Cp * 2, (cuuint64_t)g.WP2 * g.Cp * 2, (cuuint64_t)g.HP2 * g.WP2 * g.Cp * 2};
  const int kw_eff = g.fold_cf ? 1 : d->KW;               // folded: the x taps live in the channel dimension
  const int a_rows = g.a_rows;
  const cuuint32_t box[4] = {64, (cuuint32_t)a_rows, 1, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  for (int term = 0; term <= split; ++term) {
    const CUresult cr = enc(term ? &map_lo : &map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base + term * g.pack_bytes, dims, strides, box,
                            estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)cr); return B200_ERR_CUDA; }
  }
  if (!split) map_lo = map;

  static bool attr_done = false, attr_lstm_done = false;
  if (!(lstm ? attr_lstm_done : attr_done)) {
    B200_CHECK_CUDA(cudaFuncSetAttribute(lstm ? (const void*)convlstm_tma_kernel : (const void*)conv2d_tma_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, TM_SMEM_BUDGET));
    (lstm ? attr_lstm_done : attr_done) = true;
  }
  ConvTmaArgs a{};
  a.d = *d; a.w_img = reinterpret_cast<const char*>(w_images); a.bias = bias; a.res = residual; a.y = y;
  if (chain && chain->yp) {
    a.yp = chain->yp; a.yp_hp2 = chain->hp2; a.yp_wp2 = chain->wp2; a.yp_cp = chain->cp; a.yp_pad_h = chain->pad_h;
    a.yp_pad_w = chain->pad_w; a.yp_c_off = chain->c_off;
  }
  if (g.fold_cf) { a.d.KW = 1; a.d.Cin = g.fold_cf * d->KW; }
  a.OH = g.OH; a.OW = g.OW; a.x_tiles = (g.OW + 127) / 128; a.cchunks = g.cchunks; a.n_chunks = g.n_chunks;
  a.n_tile = g.n_tile; a.n_tiles_n = g.n_tiles_n; a.phases = g.phases; a.shift = g.shift;
  a.a_rows = a_rows; a.split = split;
  a.a_stage = (a_rows * 128 + 1023) / 1024 * 1024 * (1 + split);
  const int b_bytes = g.n_tile * 128 * (1 + split);
  // x taps that share one activation box are fetched as one bulk copy while that stays <= 32 KB
  const int nsub_max = (kw_eff + d->stride - 1) / d->stride;
  int b_group = 32768 / b_bytes; if (b_group < 1) b_group = 1; if (b_group > nsub_max) b_group = nsub_max;
  a.b_group = b_group; a.b_stage = b_group * b_bytes;
  // shared memory: at least 3 B stages (2 for the widest tiles), up to 6 A stages, the rest goes to the B ring;
  // narrow layers keep the whole weight image resident instead (no per-chunk weight traffic or barriers)
  const int avail = TM_SMEM_BUDGET - TM_BAR_BYTES;
  a.resident = (!split && g.n_tiles_n == 1 && (int64_t)g.n_chunks * b_bytes <= 100 * 1024) ? 1 : 0;
  int n_a, n_b;
  if (a.resident) {
    a.b_group = 1; a.b_stage = b_bytes;
    n_b = g.n_chunks;                                      // "ring" = the resident image
    n_a = (avail - n_b * a.b_stage) / a.a_stage;
    if (n_a > TM_MAX_A) n_a = TM_MAX_A;
  } else {
    n_a = (avail - 3 * a.b_stage) / a.a_stage;
    if (n_a > 6) n_a = 6;
    if (n_a < 2) n_a = 2;
    n_b = (avail - n_a * a.a_stage) / a.b_stage;
    if (n_b > TM_MAX_B) n_b = TM_MAX_B;
  }
  B200_REQUIRE(n_a >= 2 && (a.resident || n_b >= 2), "tile does not fit in shared memory");
  a.n_a = n_a; a.n_b = n_b;
  const int smem_bytes = n_a * a.a_stage + n_b * a.b_stage + TM_BAR_BYTES;
  const int64_t tiles = (int64_t)d->N * g.OH * a.x_tiles * g.n_tiles_n;
  B200_REQUIRE(tiles < (1ll << 31), "too many tiles");
  a.total_tiles = (int)tiles;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const unsigned grid = (unsigned)(tiles < sms ? tiles : sms);
  if (lstm) convlstm_tma_kernel<<<grid, TM_THREADS, smem_bytes, st>>>(a, map, map_lo, *lstm);
  else conv2d_tma_kernel<<<grid, TM_THREADS, smem_bytes, st>>>(a, map, map_lo);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace b200

namespace b200 { int launch_avgpool2(const float* x, float* y, int64_t planes, int H, int W, cudaStream_t st); }   // raft_kernels.cu
using namespace b200;

extern "C" {

int64_t b200_conv_tma_workspace_bytes(const B200ConvDesc* d) {
  TmaGeom g;
  if (tma_geometry(d, &g) != B200_OK) return -1;
  return g.pack_bytes + 256;
}

int64_t b200_conv_tma_weight_image_bytes(const B200ConvDesc* d) {
  TmaGeom g;
  if (tma_geometry(d, &g) != B200_OK) return -1;
  return (int64_t)g.n_tiles_n * g.n_chunks * g.n_tile * 128;
}

int b200_conv_tma_weight_images(const B200ConvDesc* d, const float* w, void* images, void* stream) {
  B200_REQUIRE(w && images, "null pointer");
  TmaGeom g;
  if (int rc = tma_geometry(d, &g)) return rc;
  const int KHW = d->KH * d->KW;
  return launch_weight_images(d, g, w, (int64_t)d->Cin * KHW, KHW, 1, 1.0f, 0, images, reinterpret_cast<cudaStream_t>(stream));
}

/* A convolution can consume a packed input written by its producers when its packing is the plain one: stride 1, no
 * upsampling, x taps not folded into the channel vector.  Zero padding: the halo of the buffer stays zero; reflection
 * padding: the consumer call first mirrors the interior into the halo (conv_reflect_halo_kernel). */
int b200_conv_tma_chainable(const B200ConvDesc* next) {
  TmaGeom g;
  if (!next || tma_geometry(next, &g) != B200_OK) return 0;
  return (next->stride == 1 && next->upsample == 1 && g.fold_cf == 0 && next->in_c_off == 0 &&
          next->in_c_total == next->Cin) ? 1 : 0;
}

// where the packed input of `d` lives: the caller's pre-packed buffer, or the (aligned) workspace the repack fills;
// a pre-packed input with reflection padding gets its halo mirrored here
static int tma_input_base(const B200ConvDesc* d, const TmaGeom& g, void* in_packed, void* workspace, int64_t workspace_bytes,
                          const char* who, cudaStream_t st, char** base) {
  if (in_packed) {
    B200_REQUIRE(b200_conv_tma_chainable(d), "this convolution cannot take a pre-packed input");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(in_packed) & 255) == 0, "packed input must be 256-byte aligned");
    *base = reinterpret_cast<char*>(in_packed);
    if (d->pad_mode == 1 && (d->pad_h > 0 || d->pad_w > 0)) {
      const int64_t threads = (int64_t)d->N * ((int64_t)g.HP2 * g.WP2 - (int64_t)d->H * d->W) * (g.Cp / 8);
      conv_reflect_halo_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(
          reinterpret_cast<__half*>(*base), d->N, d->H, d->W, d->pad_h, d->pad_w, g.Cp);
      B200_CHECK_LAUNCH();
    }
    return B200_OK;
  }
  B200_REQUIRE(workspace, "null workspace");
  *base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  if (*base + g.pack_bytes > reinterpret_cast<char*>(workspace) + workspace_bytes) {
    set_error("%s: workspace too small (%lld < %lld)", who, (long long)workspace_bytes, (long long)(g.pack_bytes + 256));
    return B200_ERR_WORKSPACE;
  }
  return B200_OK;
}

int b200_conv2d_tma_chain(const B200ConvDesc* d, const float* x, void* in_packed, const void* w_images, const float* bias,
                          const float* residual, float* y, void* out_packed, const B200ConvDesc* next, int32_t next_c_off,
                          void* workspace, int64_t workspace_bytes, void* stream) {
  B200_REQUIRE(d && w_images && (x || in_packed) && (y || out_packed), "null pointer");
  TmaGeom g;
  if (int rc = tma_geometry(d, &g)) return rc;
  B200_REQUIRE(d->in_c_off >= 0 && d->in_c_off + d->Cin <= d->in_c_total && d->out_c_off >= 0 &&
               d->out_c_off + d->Cout <= d->out_c_total, "channel slice out of range");
  if (residual) B200_REQUIRE(d->res_c_off >= 0 && d->res_c_off + d->Cout <= d->res_c_total, "residual slice out of range");
  if (!b200_device_supports_tc()) { set_error("b200_conv2d_tma_chain needs a compute-capability 9.x device"); return B200_ERR_UNSUPPORTED; }
  ChainOut co;
  if (out_packed) {
    B200_REQUIRE(next && b200_conv_tma_chainable(next), "the consumer convolution cannot take a pre-packed input");
    TmaGeom gn;
    if (int rc = tma_geometry(next, &gn)) return rc;
    B200_REQUIRE(next->N == d->N && next->H == g.OH && next->W == g.OW, "consumer geometry does not match this output");
    B200_REQUIRE(next_c_off >= 0 && next_c_off + d->Cout <= next->Cin && (next_c_off & 7) == 0 && (d->Cout & 7) == 0,
                 "chained channel slice must lie inside the consumer's input and be a multiple of 8 channels");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(out_packed) & 255) == 0, "packed output must be 256-byte aligned");
    co.yp = reinterpret_cast<__half*>(out_packed); co.hp2 = gn.HP2; co.wp2 = gn.WP2; co.cp = gn.Cp;
    co.pad_h = next->pad_h; co.pad_w = next->pad_w; co.c_off = next_c_off;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  char* base = nullptr;
  if (int rc = tma_input_base(d, g, in_packed, workspace, workspace_bytes, "b200_conv2d_tma_chain", st, &base)) return rc;
  return launch_conv_tma(d, g, in_packed ? nullptr : x, base, w_images, bias, residual, y, 0, 1.0f, st, &co);
}

int b200_conv_tma_pack_chain(const B200ConvDesc* next, const float* x, int32_t C, void* out_packed, int32_t next_c_off,
                             void* stream) {
  B200_REQUIRE(next && x && out_packed, "null pointer");
  B200_REQUIRE(b200_conv_tma_chainable(next), "the consumer convolution cannot take a pre-packed input");
  TmaGeom g;
  if (int rc = tma_geometry(next, &g)) return rc;
  B200_REQUIRE(C > 0 && next_c_off >= 0 && next_c_off + C <= next->Cin && (next_c_off & 7) == 0 && (C & 7) == 0,
               "packed channel slice must lie inside the consumer's input and be a multiple of 8 channels");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(out_packed) & 255) == 0, "packed output must be 256-byte aligned");
  B200_REQUIRE(g.HP2 <= 65535 && (int64_t)next->N * ((C + 63) / 64) <= 65535, "input too large for the repack grid");
  B200ConvDesc s = *next;                                 // the source tensor: C channels at the consumer's input extent
  s.Cin = C; s.in_c_total = C; s.in_c_off = 0;
  conv_pack_input_kernel<<<dim3((g.WP2 + 31) / 32, g.HP2, next->N * ((C + 63) / 64)), 256, 0,
                           reinterpret_cast<cudaStream_t>(stream)>>>(x, reinterpret_cast<__half*>(out_packed), s, g.HP2, g.WP2,
                                                                      g.Cp, 1, 1.0f, 0, 0, next_c_off, C);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// the gate convolution of a ConvLSTM: Cout = 4C (C % 8 == 0), stride 1, no upsampling / activation / scale / residual,
// the whole output (no slice)
static int lstm_geometry(const B200ConvDesc* d, TmaGeom* g) {
  if (int rc = tma_geometry(d, g)) return rc;
  B200_REQUIRE(d->Cout % 32 == 0, "ConvLSTM gates: Cout must be 4 * C with C a multiple of 8");
  B200_REQUIRE(d->stride == 1 && d->upsample == 1 && d->act == B200_ACT_NONE && d->out_scale == 1.0f &&
               d->out_c_off == 0 && d->out_c_total == d->Cout && d->res_c_total == 0 && d->res_c_off == 0,
               "ConvLSTM gates: stride 1, no upsampling, activation, output scale, output slice or residual");
  return B200_OK;
}

int b200_convlstm_tma_weight_images(const B200ConvDesc* d, const float* w, void* images, void* stream) {
  B200_REQUIRE(w && images, "null pointer");
  TmaGeom g;
  if (int rc = lstm_geometry(d, &g)) return rc;
  const int KHW = d->KH * d->KW;
  return launch_weight_images(d, g, w, (int64_t)d->Cin * KHW, KHW, 1, 1.0f, 0, images, reinterpret_cast<cudaStream_t>(stream),
                              d->Cout / 4);
}

int b200_convlstm_tma(const B200ConvDesc* d, const float* x, void* in_packed, const void* w_images, const float* bias,
                      const float* prev_cell, float* hidden, float* cell, void* workspace, int64_t workspace_bytes,
                      void* stream) {
  B200_REQUIRE(d && w_images && (x || in_packed) && hidden, "null pointer");
  TmaGeom g;
  if (int rc = lstm_geometry(d, &g)) return rc;
  B200_REQUIRE(d->in_c_off >= 0 && d->in_c_off + d->Cin <= d->in_c_total, "channel slice out of range");
  if (!b200_device_supports_tc()) { set_error("b200_convlstm_tma needs a compute-capability 9.x device"); return B200_ERR_UNSUPPORTED; }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  char* base = nullptr;
  if (int rc = tma_input_base(d, g, in_packed, workspace, workspace_bytes, "b200_convlstm_tma", st, &base)) return rc;
  const LstmArgs l{prev_cell, hidden, cell, d->Cout / 4};
  return launch_conv_tma(d, g, in_packed ? nullptr : x, base, w_images, bias, nullptr, nullptr, 0, 1.0f, st, nullptr, &l);
}

/* ---- all-pairs correlation (RAFT CorrBlock level 0, src/models/stage_1/core/corr.py:56-64) as a 1x1 "convolution":
 * input = fmap2 (pixels p2), weights[co = p1][ci] = fmap1[ci][p1], output [p1][p2].  The reference computes it in
 * fp32 (fmaps are cast with .float() and TF32 matmul is off by default), so both operands are split into
 * (hi, lo) fp16 pairs, pre-scaled by 2^4: 3 tensor-core products per element, fp32 accumulation — the same
 * fp32-grade emulation as the stage-1 MLPs. */
static void corr_desc(int dim, int H8, int W8, B200ConvDesc* d) {
  *d = B200ConvDesc{};
  d->N = 1; d->Cin = dim; d->H = H8; d->W = W8; d->in_c_total = dim; d->in_c_off = 0;
  d->Cout = H8 * W8; d->KH = 1; d->KW = 1; d->stride = 1; d->pad_h = 0; d->pad_w = 0; d->pad_mode = 0; d->upsample = 1;
  d->out_c_total = H8 * W8; d->out_c_off = 0; d->act = 0;
  d->out_scale = 1.0f / sqrtf((float)dim) / 256.0f;       // undo the two 2^4 operand scales
  d->res_c_total = 0; d->res_c_off = 0;
}

// floats of the three pooled copies of fmap2 (levels 1..3 of the pyramid are GEMMs on them, see below)
static int64_t corr_pooled_floats(int dim, int H8, int W8) {
  int64_t n = 0;
  int h = H8, w = W8;
  for (int l = 1; l < 4; ++l) { h /= 2; w /= 2; n += (int64_t)dim * h * w + 64; }
  return n;
}

int64_t b200_corr_build_tc_workspace_bytes(int32_t dim, int32_t H8, int32_t W8) {
  if (dim <= 0 || H8 < 8 || W8 < 8) return -1;
  B200ConvDesc d; corr_desc(dim, H8, W8, &d);
  TmaGeom g;
  if (tma_geometry(&d, &g) != B200_OK) return -1;
  return 2 * g.pack_bytes + 2 * (int64_t)g.n_tiles_n * g.n_chunks * g.n_tile * 128 + corr_pooled_floats(dim, H8, W8) * 4 + 2048;
}

int64_t b200_corr_build_tc_batch_workspace_bytes(int32_t batch, int32_t dim, int32_t H8, int32_t W8) {
  return batch >= 1 ? b200_corr_build_tc_workspace_bytes(dim, H8, W8) : -1;   // the samples reuse one workspace
}

int b200_corr_build_tc(const float* fmap1, const float* fmap2, int32_t dim, int32_t H8, int32_t W8, float* pyramid,
                       void* workspace, int64_t workspace_bytes, void* stream) {
  return b200_corr_build_tc_batch(fmap1, fmap2, 1, dim, H8, W8, pyramid, workspace, workspace_bytes, stream);
}

// B pairs, one after the other in one workspace (stream order serialises them): each sample's fmap1 becomes its own
// weight images, so a sample's launches are exactly the single-pair ones and conv2d_tma_kernel is not re-instantiated.
// At 640x360 one sample's level-0 GEMM already fills the device (~675 tiles).
int b200_corr_build_tc_batch(const float* fmap1, const float* fmap2, int32_t batch, int32_t dim, int32_t H8, int32_t W8,
                             float* pyramid, void* workspace, int64_t workspace_bytes, void* stream) {
  B200_REQUIRE(fmap1 && fmap2 && pyramid && workspace && batch >= 1 && dim > 0 && H8 >= 8 && W8 >= 8, "bad arguments");
  if (!b200_device_supports_tc()) { set_error("b200_corr_build_tc needs a compute-capability 9.x device"); return B200_ERR_UNSUPPORTED; }
  B200ConvDesc d; corr_desc(dim, H8, W8, &d);
  TmaGeom g;
  if (int rc = tma_geometry(&d, &g)) return rc;
  const int64_t need = b200_corr_build_tc_workspace_bytes(dim, H8, W8);
  B200_REQUIRE(workspace_bytes >= need, "b200_corr_build_tc: workspace too small");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~(uintptr_t)255);
  char* images = base + 2 * g.pack_bytes;                  // pack_bytes is a multiple of 128
  const int HW = H8 * W8;
  const int64_t fmap_floats = (int64_t)dim * HW, pyr_floats = b200_corr_pyramid_floats(H8, W8);
  const int64_t image_bytes = 2 * (int64_t)g.n_tiles_n * g.n_chunks * g.n_tile * 128;
  for (int b = 0; b < batch; ++b) {
    const float* f1 = fmap1 + b * fmap_floats;
    const float* f2 = fmap2 + b * fmap_floats;
    float* pyr = pyramid + b * pyr_floats;
    if (int rc = launch_weight_images(&d, g, f1, /*co*/ 1, /*ci*/ HW, /*tap*/ 0, 16.0f, 1, images, st)) return rc;
    if (int rc = launch_conv_tma(&d, g, f2, base, images, nullptr, nullptr, pyr, 1, 16.0f, st)) return rc;
    // Levels 1..3 (corr.py:27-31: avg_pool2d of the previous level over the TARGET pixel grid).  Average pooling is
    // linear in fmap2, so level l = fmap1^T . avgpool^l(fmap2): three small GEMMs on pooled 33 MB feature maps with the
    // same fmap1 weight images, instead of three passes that re-read the 4.2 GB level-0 volume (1.7 of 3.5 ms at 1080p).
    float* pooled = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(images + image_bytes) + 255) & ~(uintptr_t)255);
    const float* src = f2;
    float* out = pyr + (int64_t)HW * HW;
    int h = H8, w = W8;
    for (int l = 1; l < 4; ++l) {
      if (int rc = launch_avgpool2(src, pooled, dim, h, w, st)) return rc;
      h /= 2; w /= 2;
      if (h < 1 || w < 1) break;
      B200ConvDesc dl = d;
      dl.H = h; dl.W = w;                                   // queries (output channels) stay at full resolution
      TmaGeom gl;
      if (int rc = tma_geometry(&dl, &gl)) return rc;
      if (int rc = launch_conv_tma(&dl, gl, pooled, base, images, nullptr, nullptr, out, 1, 16.0f, st)) return rc;
      out += (int64_t)HW * h * w;
      src = pooled;
      pooled += (((int64_t)dim * h * w + 63) / 64) * 64;
    }
  }
  return B200_OK;
}

}  // extern "C"
