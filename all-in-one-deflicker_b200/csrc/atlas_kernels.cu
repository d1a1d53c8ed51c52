// Non-GEMM kernels of the stage-1 atlas loop: video repacking, sample selection / gather, positional
// encoding forward/backward, the fused loss head, Adam, render helpers.
// Reference lines restated are cited per kernel (paths relative to the reference root).
#include "atlas_internal.cuh"
#include "loss_math.h"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// video repack: reference layouts (T innermost, unwrap_utils.py:112-122) -> frame-major records
// ---------------------------------------------------------------------------------------------
__global__ void video_pack_kernel(const float* __restrict__ fr, const float* __restrict__ dx,
                                  const float* __restrict__ dy, const float* __restrict__ ff,
                                  const float* __restrict__ fb, const float* __restrict__ mf,
                                  const float* __restrict__ mb, int H, int W, int T, int t_begin, int t_end,
                                  float* __restrict__ rec) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;     // local pixel index
  const int64_t HW = (int64_t)H * W;
  if (p >= HW * (t_end - t_begin)) return;
  const int t = (int)(p / HW) + t_begin;
  const int64_t yx = p % HW;                                            // y*W + x
  float4 r[4];
  float v[16];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    v[c] = fr[(yx * 3 + c) * T + t];
    v[3 + c] = dx[(yx * 3 + c) * T + t];
    v[6 + c] = dy[(yx * 3 + c) * T + t];
  }
  v[9] = ff[(yx * 2 + 0) * T + t];  v[10] = ff[(yx * 2 + 1) * T + t];
  v[11] = fb[(yx * 2 + 0) * T + t]; v[12] = fb[(yx * 2 + 1) * T + t];
  v[13] = mf[yx * T + t];           v[14] = mb[yx * T + t];
  v[15] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) r[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  float4* dst = reinterpret_cast<float4*>(rec + p * B200_RECORD_FLOATS);
#pragma unroll
  for (int q = 0; q < 4; ++q) dst[q] = r[q];
}

// bit n of the bitmap <=> mask value of pixel-table entry n = (t*H + y)*W + x is non-zero
__global__ void mask_bits_kernel(const float* __restrict__ mf, const float* __restrict__ mb, int H, int W,
                                 int T, uint32_t* __restrict__ bits_f, uint32_t* __restrict__ bits_b) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t HW = (int64_t)H * W, N = HW * T;
  bool f = false, b = false;
  if (n < N) {
    const int64_t t = n / HW, yx = n % HW;
    f = mf[yx * T + t] != 0.f;
    b = mb[yx * T + t] != 0.f;
  }
  const uint32_t wf = __ballot_sync(0xffffffffu, f), wb = __ballot_sync(0xffffffffu, b);
  if ((threadIdx.x & 31) == 0 && n < N) { bits_f[n >> 5] = wf; bits_b[n >> 5] = wb; }
}

int launch_video_pack(const float* fr, const float* dx, const float* dy, const float* ff, const float* fb,
                      const float* mf, const float* mb, int H, int W, int T, int t_begin, int t_end,
                      float* rec, uint32_t* bits_f, uint32_t* bits_b, cudaStream_t st) {
  const int64_t n_local = (int64_t)H * W * (t_end - t_begin);
  if (n_local > 0) {
    video_pack_kernel<<<(unsigned)((n_local + 255) / 256), 256, 0, st>>>(fr, dx, dy, ff, fb, mf, mb, H, W, T,
                                                                           t_begin, t_end, rec);
    B200_CHECK_LAUNCH();
  }
  const int64_t N = (int64_t)H * W * T;
  mask_bits_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(mf, mb, H, W, T, bits_f, bits_b);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------
// sampling: selection of the resident samples, record gather, coordinate rows.  One thread per sample of the
// GLOBAL batch.  src/stage1_neural_atlas.py:159-171 (jif_all[:, inds], rgb gather, xyt), loss_utils.py:138-151
// (x+1 / y+1 rows, dx/dy gather), :230-233 (rigidity rows), :326-351 (flow-matched rows and the torch.where counts).
//
// counters (zeroed by a memset node before the launch):
//   [0] n_local   samples whose frame is resident here (slot order: batch order on one GPU; claimed with a
//                 warp-aggregated atomic when frame-sharded — the order only permutes fp32 summation)
//   [1] n_fwd     [2] n_bwd    valid forward / backward flow rows of the WHOLE batch (from the replicated
//                 bitmaps): the denominators of the two flow means on every rank
//   [3] [4]       gradient-scale bits of the tensor-core path (written by the loss head)
//   [5] n_lf      [6] n_lb     resident valid flow rows: the flow-match groups are COMPACTED to these counts
//                 (row p of group G_FWD belongs to the sample whose target row stores p+1), so the networks are
//                 never evaluated on rows the reference's torch.where drops
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int warp_claim(bool take, int* counter, int lane) {
  const uint32_t m = __ballot_sync(0xffffffffu, take);
  int base = 0;
  if (m) {
    const int leader = __ffs(m) - 1;
    if (lane == leader) base = atomicAdd(counter, __popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
  }
  return base + __popc(m & ((1u << lane) - 1u));
}

template <bool ALL_LOCAL>
__global__ void sample_kernel(const int64_t* __restrict__ indices, int* __restrict__ counters, B200Video vid,
                              SampleGeom geo, int cap, int batch, int n_groups, const float* __restrict__ matte,
                              float4* __restrict__ x_map, float* __restrict__ targets) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;      // index into the global batch (or a padding slot)
  const int lane = threadIdx.x & 31;
  bool local = false, wf = false, wb = false, gf = false, gb = false;
  int t = 0, y = 0, x = 0;
  float v[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) v[q] = 0.f;
  if (b < batch) {
    const int64_t n = indices[b];
    const int64_t HW = (int64_t)vid.H * vid.W;
    t = (int)(n / HW);
    y = (int)((n / vid.W) % vid.H);
    x = (int)(n % vid.W);
    local = ALL_LOCAL || (t >= vid.t_begin && t < vid.t_end);
    if (local) {
      const float4* rec = reinterpret_cast<const float4*>(
          vid.records + (((int64_t)(t - vid.t_begin) * vid.H + y) * vid.W + x) * B200_RECORD_FLOATS);
      const float4 r0 = __ldg(rec), r1 = __ldg(rec + 1), r2 = __ldg(rec + 2), r3 = __ldg(rec + 3);
      v[0] = r0.x; v[1] = r0.y; v[2] = r0.z; v[3] = r0.w; v[4] = r1.x; v[5] = r1.y; v[6] = r1.z; v[7] = r1.w;
      v[8] = r2.x; v[9] = r2.y; v[10] = r2.z; v[11] = r2.w; v[12] = r3.x; v[13] = r3.y; v[14] = r3.z; v[15] = r3.w;
      wf = v[13] != 0.f; wb = v[14] != 0.f;
    }
    if (ALL_LOCAL) { gf = wf; gb = wb; }
    else {
      gf = (vid.mask_fwd_bits[n >> 5] >> (n & 31)) & 1u;
      gb = (vid.mask_bwd_bits[n >> 5] >> (n & 31)) & 1u;
    }
  }
  // whole-batch flow counts, slot of this sample, slots of its two flow-matched rows
  {
    const uint32_t mf = __ballot_sync(0xffffffffu, gf), mb = __ballot_sync(0xffffffffu, gb);
    if (lane == 0) {
      if (mf) atomicAdd(counters + 1, __popc(mf));
      if (mb) atomicAdd(counters + 2, __popc(mb));
    }
  }
  int s = b;
  if (!ALL_LOCAL) s = warp_claim(local, counters + 0, lane);
  const int pf = warp_claim(local && wf, counters + 5, lane);
  const int pb = warp_claim(local && wb, counters + 6, lane);
  if (ALL_LOCAL && b == 0) counters[0] = batch;
  if (local) {
    const float fx = (float)x, fy = (float)y, ft = (float)t;
    const float hL = geo.half_larger, hX = geo.half_resx, hT = geo.half_frames;
    const float tn = norm_coord(ft, hT);
    float4 rows[G_COUNT];
    rows[G_BASE] = make_float4(norm_coord(fx, hL), norm_coord(fy, hL), tn, 0.f);
    rows[G_XP1] = make_float4(norm_coord(fx + 1.f, hX), norm_coord(fy, hX), tn, 0.f);
    rows[G_YP1] = make_float4(norm_coord(fx, hX), norm_coord(fy + 1.f, hX), tn, 0.f);
    rows[G_YMD] = make_float4(norm_coord(fx, hL), norm_coord(fy - geo.d_local, hL), tn, 0.f);
    rows[G_XMD] = make_float4(norm_coord(fx - geo.d_local, hL), norm_coord(fy, hL), tn, 0.f);
    rows[G_FWD] = make_float4(norm_coord(__fadd_rn(fx, v[9]), hL), norm_coord(__fadd_rn(fy, v[10]), hL),
                              norm_coord(ft + 1.f, hT), 0.f);
    rows[G_BWD] = make_float4(norm_coord(__fadd_rn(fx, v[11]), hL), norm_coord(__fadd_rn(fy, v[12]), hL),
                              norm_coord(ft - 1.f, hT), 0.f);
    rows[G_YMG] = make_float4(norm_coord(fx, hL), norm_coord(fy - geo.d_global, hL), tn, 0.f);
    rows[G_XMG] = make_float4(norm_coord(fx - geo.d_global, hL), norm_coord(fy, hL), tn, 0.f);
#pragma unroll
    for (int g = 0; g < G_COUNT; ++g) {
      if (g >= n_groups) continue;
      if (g == G_FWD) { if (wf) x_map[(int64_t)g * cap + pf] = rows[g]; }
      else if (g == G_BWD) { if (wb) x_map[(int64_t)g * cap + pb] = rows[g]; }
      else x_map[(int64_t)g * cap + s] = rows[g];
    }
    float4* tdst = reinterpret_cast<float4*>(targets + (int64_t)s * TARGET_FLOATS);
    tdst[0] = make_float4(v[0], v[1], v[2], v[3]);
    tdst[1] = make_float4(v[4], v[5], v[6], v[7]);
    // column 11: the sample's matte value, which travels with its slot (slot order is not batch order on a shard)
    const float a_gt = matte ? matte[((int64_t)(t - vid.t_begin) * vid.H + y) * vid.W + x] : 0.f;
    tdst[2] = make_float4(v[8], wf ? (float)(pf + 1) : 0.f, wb ? (float)(pb + 1) : 0.f, a_gt);
  } else if (ALL_LOCAL && b < cap) {
    // padding slots of the last tile: finite rows, zero targets
#pragma unroll
    for (int g = 0; g < G_COUNT; ++g)
      if (g < n_groups && g != G_FWD && g != G_BWD) x_map[(int64_t)g * cap + b] = make_float4(0.f, 0.f, 0.f, 0.f);
    float4* tdst = reinterpret_cast<float4*>(targets + (int64_t)b * TARGET_FLOATS);
    tdst[0] = tdst[1] = tdst[2] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

int launch_select_sample(const int64_t* indices, int B, const B200Video& vid, const SampleGeom& geo, int cap,
                         int n_groups, int* counters, int* list, float* x_map, float* targets,
                         cudaStream_t st, const float* matte) {
  (void)list;
  B200_CHECK_CUDA(cudaMemsetAsync(counters, 0, 32, st));
  if (vid.t_begin == 0 && vid.t_end == vid.T)
    sample_kernel<true><<<(cap + 127) / 128, 128, 0, st>>>(indices, counters, vid, geo, cap, B, n_groups, matte,
                                                            reinterpret_cast<float4*>(x_map), targets);
  else
    sample_kernel<false><<<(B + 127) / 128, 128, 0, st>>>(indices, counters, vid, geo, cap, B, n_groups, matte,
                                                           reinterpret_cast<float4*>(x_map), targets);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// pre_train_mapping rows (unwrap_utils.py:183-190): every slot is valid; counters[0] = B
__global__ void pretrain_sample_kernel(const int64_t* __restrict__ ys, const int64_t* __restrict__ xs, int B,
                                       int cap, float half_larger, float t_norm, float4* __restrict__ x_map,
                                       int* __restrict__ counters) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s == 0) { counters[0] = B; counters[3] = 0; counters[4] = 0; counters[5] = 0; counters[6] = 0; }
  if (s >= cap) return;
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if (s < B) r = make_float4(norm_coord((float)xs[s], half_larger), norm_coord((float)ys[s], half_larger), t_norm, 0.f);
  x_map[s] = r;
}

__device__ __forceinline__ void publish_gmax(float mx, int* gmax_bits) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0 && mx > 0.f) atomicMax(gmax_bits, __float_as_int(mx));
}

__global__ void pretrain_loss_kernel(const float4* __restrict__ x_map, const float* __restrict__ uv, int B,
                                     int cap, float uv_scale, float* __restrict__ d_uv,
                                     float* __restrict__ losses, int* __restrict__ gmax_bits) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  float val = 0.f;
  if (s < cap) {
    float g[2] = {0.f, 0.f};
    if (s < B) {
      const float4 x = x_map[s];
      const float u[2] = {uv[2 * s], uv[2 * s + 1]};
      val = pretrain_term(x.x, x.y, u, uv_scale, 1.0f / (float)B, g);
    }
    d_uv[2 * s] = g[0];
    d_uv[2 * s + 1] = g[1];
    publish_gmax(fmaxf(fabsf(g[0]), fabsf(g[1])), gmax_bits);
  } else {
    publish_gmax(0.f, gmax_bits);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) val += __shfl_xor_sync(0xffffffffu, val, o);
  if ((threadIdx.x & 31) == 0 && val != 0.f) atomicAdd(losses, val / (float)B);
}

int launch_pretrain_sample(const int64_t* ys, const int64_t* xs, int B, int cap, float half_larger,
                           float t_norm, float* x_map, int* counters, cudaStream_t st) {
  pretrain_sample_kernel<<<(cap + 127) / 128, 128, 0, st>>>(ys, xs, B, cap, half_larger, t_norm,
                                                             reinterpret_cast<float4*>(x_map), counters);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int launch_pretrain_loss(const float* x_map, const float* uv, int B, int cap, float uv_scale, float* d_uv,
                         float* losses, int* counters, cudaStream_t st) {
  pretrain_loss_kernel<<<(cap + 127) / 128, 128, 0, st>>>(reinterpret_cast<const float4*>(x_map), uv, B, cap,
                                                           uv_scale, d_uv, losses, counters + 4);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------
// positional encoding (implicit_neural_networks.py:9-13) of in = x*scale + shift.
// One thread per (row, frequency).  Written to the layer-0 input and to the skip slots.
// ---------------------------------------------------------------------------------------------
struct PeTargets {
  float* out[4];
  int ld[4];
  int col[4];
  int n;
};

__device__ __forceinline__ bool row_is_live(int64_t row, int64_t cap, const int* n_valid) {
  if (n_valid == nullptr || cap <= 0) return true;
  // whole 128-row tiles that contain at least one valid row are processed
  const int lim = (*n_valid + kTileRows - 1) / kTileRows * kTileRows;
  return (row % cap) < lim;
}

__global__ void pe_forward_kernel(const float* __restrict__ x, int ldx, float scale, float shift, int in_dim,
                                  int freqs, PeTargets tg, int64_t rows, int64_t cap,
                                  const int* __restrict__ n_valid) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t row = e / freqs;
  const int k = (int)(e % freqs);
  if (row >= rows || !row_is_live(row, cap, n_valid)) return;
  const float bk = pe_freq(k);
  for (int j = 0; j < in_dim; ++j) {
    const float v = x[row * ldx + j] * scale + shift;
    const float arg = v * bk;
    const float sv = sinf(arg), cv = cosf(arg);
    for (int q = 0; q < tg.n; ++q) {
      float* o = tg.out[q] + row * tg.ld[q] + tg.col[q] + k * 2 * in_dim;
      o[j] = sv;
      o[in_dim + j] = cv;
    }
  }
}

int launch_pe_forward(const float* x, int ldx, float scale, float shift, int in_dim, int freqs,
                      float* out0, int ld0, float* const* skip_outs, const int* skip_lds, int n_skip,
                      int skip_col, const RowSpan& span, cudaStream_t st) {
  PeTargets tg{};
  tg.out[0] = out0; tg.ld[0] = ld0; tg.col[0] = 0; tg.n = 1;
  for (int i = 0; i < n_skip && tg.n < 4; ++i) {
    tg.out[tg.n] = skip_outs[i]; tg.ld[tg.n] = skip_lds[i]; tg.col[tg.n] = skip_col; ++tg.n;
  }
  if (n_skip > 3) { set_error("at most 3 skip layers supported"); return B200_ERR_UNSUPPORTED; }
  const int64_t total = span.rows * freqs;
  pe_forward_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, ldx, scale, shift, in_dim, freqs, tg,
                                                                      span.rows, span.cap, span.n_valid);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// d in_j = sum_k b_k (dsin_kj * cos_kj - dcos_kj * sin_kj);  d x = scale * d in
__global__ void pe_backward_kernel(const float* __restrict__ pe, int ld_pe, const float* __restrict__ dpe,
                                   int ld_dpe, int in_dim, int freqs, float scale, float* __restrict__ dx,
                                   int ld_dx, int accumulate, int64_t rows, int64_t cap,
                                   const int* __restrict__ n_valid) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t row = e / in_dim;
  const int j = (int)(e % in_dim);
  if (row >= rows || !row_is_live(row, cap, n_valid)) return;
  float acc = 0.f;
  for (int k = 0; k < freqs; ++k) {
    const int base = k * 2 * in_dim;
    const float s = pe[row * ld_pe + base + j], c = pe[row * ld_pe + base + in_dim + j];
    const float ds = dpe[row * ld_dpe + base + j], dc = dpe[row * ld_dpe + base + in_dim + j];
    acc += pe_freq(k) * (ds * c - dc * s);
  }
  float* o = dx + row * ld_dx + j;
  if (accumulate) *o += scale * acc; else *o = scale * acc;
}

int launch_pe_backward(const float* pe, int ld_pe, const float* dpe, int ld_dpe, int in_dim, int freqs,
                       float scale, float* d_x, int ld_dx, int accumulate, const RowSpan& span,
                       cudaStream_t st) {
  const int64_t total = span.rows * in_dim;
  pe_backward_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(pe, ld_pe, dpe, ld_dpe, in_dim, freqs,
                                                                       scale, d_x, ld_dx, accumulate, span.rows,
                                                                       span.cap, span.n_valid);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------
// fused loss head: one thread per sample slot (loss_math.h).  Writes d/d uv for all mapping rows,
// d/d y for the atlas rows and accumulates the loss vector.
// ---------------------------------------------------------------------------------------------
__global__ void loss_kernel(const float* __restrict__ uv, const float* __restrict__ y_atlas,
                            const float* __restrict__ targets, int* __restrict__ counters, int cap,
                            int n_groups, LossConfig cfg, float* __restrict__ d_uv, float* __restrict__ d_y,
                            float* __restrict__ losses) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_local = counters[0], n_f = counters[1], n_b = counters[2], n_lf = counters[5], n_lb = counters[6];
  cfg.inv_nf = n_f > 0 ? 1.0f / (float)n_f : 0.f;
  cfg.inv_nb = n_b > 0 ? 1.0f / (float)n_b : 0.f;
  float part[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float gmx = 0.f, gmy = 0.f;
  if (s < cap) {
    SampleOut out;
    int pf = -1, pb = -1;                 // compacted rows of this sample in the two flow-match groups
    if (s < n_local) {
      SampleIn in;
      const float* tg = targets + (int64_t)s * TARGET_FLOATS;
      pf = (int)tg[9] - 1; pb = (int)tg[10] - 1;
#pragma unroll
      for (int g = 0; g < G_COUNT; ++g) {
        const int r = g == G_FWD ? pf : (g == G_BWD ? pb : s);
        if (g < n_groups && r >= 0) {
          const float2 v = *reinterpret_cast<const float2*>(uv + ((int64_t)g * cap + r) * 2);
          in.uv[g][0] = v.x; in.uv[g][1] = v.y;
        } else { in.uv[g][0] = in.uv[g][1] = 0.f; }
      }
#pragma unroll
      for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int c = 0; c < 3; ++c) in.y[g][c] = y_atlas[((int64_t)g * cap + s) * 3 + c];
#pragma unroll
      for (int c = 0; c < 3; ++c) { in.rgb[c] = tg[c]; in.dx[c] = tg[3 + c]; in.dy[c] = tg[6 + c]; }
      in.wf = pf >= 0 ? 1.f : 0.f; in.wb = pb >= 0 ? 1.f : 0.f;
      sample_loss(in, cfg, out);
      part[0] = out.rgb; part[1] = out.grad; part[2] = out.rig; part[3] = out.rig_global;
      part[4] = out.flow_f; part[5] = out.flow_b;
    } else {
#pragma unroll
      for (int g = 0; g < G_COUNT; ++g) out.duv[g][0] = out.duv[g][1] = 0.f;
#pragma unroll
      for (int g = 0; g < 3; ++g)
#pragma unroll
        for (int c = 0; c < 3; ++c) out.dy[g][c] = 0.f;
    }
#pragma unroll
    for (int g = 0; g < G_COUNT; ++g)
      if (g < n_groups) {
        if (g == G_FWD || g == G_BWD) {
          // this sample's compacted row, and (as slot owner) zero for the padding rows of the group's last tile
          const int r = g == G_FWD ? pf : pb, n_rows = g == G_FWD ? n_lf : n_lb;
          if (r >= 0) *reinterpret_cast<float2*>(d_uv + ((int64_t)g * cap + r) * 2) = make_float2(out.duv[g][0], out.duv[g][1]);
          if (s >= n_rows) *reinterpret_cast<float2*>(d_uv + ((int64_t)g * cap + s) * 2) = make_float2(0.f, 0.f);
        } else {
          *reinterpret_cast<float2*>(d_uv + ((int64_t)g * cap + s) * 2) = make_float2(out.duv[g][0], out.duv[g][1]);
        }
        gmx = fmaxf(gmx, fmaxf(fabsf(out.duv[g][0]), fabsf(out.duv[g][1])));
      }
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
      for (int c = 0; c < 3; ++c) gmy = fmaxf(gmy, fabsf(out.dy[g][c]));
#pragma unroll
    for (int g = 0; g < 3; ++g)
#pragma unroll
      for (int c = 0; c < 3; ++c) d_y[((int64_t)g * cap + s) * 3 + c] = out.dy[g][c];
  }
  // scales of this iteration's gradients for the tensor-core path: [3] atlas (dL/drgb), [4] mapping (dL/duv,
  // completed by the atlas backward)
  publish_gmax(gmy, counters + 3);
  publish_gmax(gmx, counters + 4);
  // block reduction of the six partial sums -> atomics on the loss vector
  __shared__ float red[6][8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < 6; ++q) {
    float v = part[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[q][wid] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t[6];
    for (int q = 0; q < 6; ++q) {
      float v = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += red[q][w];
      t[q] = v;
    }
    const float l_rgb = t[0] * cfg.inv_batch, l_grad = t[1] * cfg.inv_batch;
    const float l_rig = t[2] * cfg.inv_batch, l_rigg = t[3] * cfg.inv_batch;
    float l_flow = 0.5f * (t[4] * cfg.inv_nf + t[5] * cfg.inv_nb);
    // the mean over an empty set is NaN in the reference (loss value only; gradients stay finite)
    if (blockIdx.x == 0 && (n_f == 0 || n_b == 0) && cfg.inv_batch > 0.f) l_flow = nanf("");
    atomicAdd(losses + 1, l_rgb);
    atomicAdd(losses + 2, l_grad);
    atomicAdd(losses + 3, l_rig);
    atomicAdd(losses + 4, l_rigg);
    atomicAdd(losses + 5, l_flow);
    atomicAdd(losses + 0, cfg.c_rig * l_rig + cfg.c_rig_global * l_rigg + cfg.c_rgb * l_rgb +
                              cfg.c_flow * l_flow + cfg.c_grad * l_grad);
    if (blockIdx.x == 0) { losses[6] = (float)n_f; losses[7] = (float)n_b; }
  }
}

int launch_loss(const float* uv, const float* y_atlas, const float* targets, int* counters, int cap,
                int n_groups, const LossConfig& cfg, float* d_uv, float* d_y, float* losses,
                cudaStream_t st) {
  loss_kernel<<<(cap + 127) / 128, 128, 0, st>>>(uv, y_atlas, targets, counters, cap, n_groups, cfg, d_uv, d_y,
                                                  losses);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Adam (torch.optim.Adam defaults: no weight decay, no amsgrad), src/stage1_neural_atlas.py:132-134.
// Arithmetic order of torch's single-tensor implementation (_single_tensor_adam):
//   m.lerp_(g, 1-b1);  v.mul_(b2).addcmul_(g, g, value=1-b2);
//   denom = sqrt(v) / sqrt(1-b2^t) + eps;  p.addcdiv_(m, denom, value=-lr/(1-b1^t))
// ---------------------------------------------------------------------------------------------
__device__ unsigned int g_adam_ticket = 0u;

__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, int64_t n, double lr, double b1d, double b2d, double epsd,
                            float grad_scale, int64_t* __restrict__ step_in) {
  __shared__ float s_step_size, s_bc2_sqrt;
  if (threadIdx.x == 0) {
    const double t = (double)(*step_in + 1);
    const double bc1 = 1.0 - pow(b1d, t);
    const double bc2 = 1.0 - pow(b2d, t);
    s_step_size = (float)(lr / bc1);
    s_bc2_sqrt = (float)sqrt(bc2);
  }
  __syncthreads();
  const float step_size = s_step_size, bc2_sqrt = s_bc2_sqrt;
  // python floats (doubles) rounded to fp32 where torch passes them to fp32 kernels
  const float w1 = (float)(1.0 - b1d), w2 = (float)(1.0 - b2d), b2 = (float)b2d, eps = (float)epsd;
  const int64_t i4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) {
  } else if (i4 + 3 < n) {
    const float4 gg = *reinterpret_cast<const float4*>(g + i4);
    float4 pp = *reinterpret_cast<float4*>(p + i4);
    float4 mm = *reinterpret_cast<float4*>(m + i4);
    float4 vv = *reinterpret_cast<float4*>(v + i4);
    const float ga[4] = {gg.x * grad_scale, gg.y * grad_scale, gg.z * grad_scale, gg.w * grad_scale};
    float pa[4] = {pp.x, pp.y, pp.z, pp.w}, ma[4] = {mm.x, mm.y, mm.z, mm.w}, va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      ma[q] = ma[q] + w1 * (ga[q] - ma[q]);
      va[q] = va[q] * b2 + (w2 * ga[q]) * ga[q];
      const float denom = sqrtf(va[q]) / bc2_sqrt + eps;
      pa[q] = pa[q] + (-step_size * ma[q]) / denom;
    }
    *reinterpret_cast<float4*>(p + i4) = make_float4(pa[0], pa[1], pa[2], pa[3]);
    *reinterpret_cast<float4*>(m + i4) = make_float4(ma[0], ma[1], ma[2], ma[3]);
    *reinterpret_cast<float4*>(v + i4) = make_float4(va[0], va[1], va[2], va[3]);
  } else {
    for (int64_t i = i4; i < n; ++i) {
      const float gq = g[i] * grad_scale;
      const float mq = m[i] + w1 * (gq - m[i]);
      const float vq = v[i] * b2 + (w2 * gq) * gq;
      const float denom = sqrtf(vq) / bc2_sqrt + eps;
      p[i] = p[i] + (-step_size * mq) / denom;
      m[i] = mq; v[i] = vq;
    }
  }
  // the step counter is advanced by the LAST block to finish: every block has read it before taking its ticket
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&g_adam_ticket, 1u) == gridDim.x - 1) {
      *step_in += 1;
      g_adam_ticket = 0u;
    }
  }
}

int launch_adam(float* p, const float* g, float* m, float* v, int64_t n, double lr, double b1, double b2,
                double eps, float grad_scale, int64_t* step, cudaStream_t st) {
  const int64_t threads = (n + 3) / 4;
  timer_begin(TAG_ADAM, st);
  adam_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(p, g, m, v, n, lr, b1, b2, eps, grad_scale, step);
  timer_end(TAG_ADAM, st);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------
// render helpers (src/models/stage_1/evaluate.py:644-666,733)
// ---------------------------------------------------------------------------------------------
__global__ void render_rows_kernel(int W, float half_larger, float t_norm, int64_t pix_begin, int64_t count,
                                   int64_t rows_padded, float4* __restrict__ x_map) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= rows_padded) return;
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if (s < count) {
    const int64_t p = pix_begin + s;
    r = make_float4(norm_coord((float)(p % W), half_larger), norm_coord((float)(p / W), half_larger), t_norm, 0.f);
  }
  x_map[s] = r;
}

__global__ void render_out_kernel(const float* __restrict__ y, int64_t count, float* __restrict__ rgb,
                                  uint8_t* __restrict__ u8) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count * 3) return;
  const float o = (y[i] + 1.0f) * 0.5f;
  if (rgb) rgb[i] = o;
  if (u8) u8[i] = (uint8_t)(int)((double)o * 255.0);      // float64 product, truncation (evaluate.py:733)
}

int launch_render_rows(int W, float half_larger, float t_norm, int64_t pix_begin, int64_t count,
                       int64_t rows_padded, float* x_map, cudaStream_t st) {
  render_rows_kernel<<<(unsigned)((rows_padded + 255) / 256), 256, 0, st>>>(
      W, half_larger, t_norm, pix_begin, count, rows_padded, reinterpret_cast<float4*>(x_map));
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int launch_render_out(const float* y, int64_t count, float* rgb, uint8_t* u8, cudaStream_t st) {
  render_out_kernel<<<(unsigned)((count * 3 + 255) / 256), 256, 0, st>>>(y, count, rgb, u8);
  B200_CHECK_LAUNCH();
  return B200_OK;
}


// ---------------------------------------------------------------------------------------------
// helpers of the stand-alone tensor-core IMLP entry points (c_api.cu): zero-padded row packing, max |x|
// ---------------------------------------------------------------------------------------------
__global__ void pack_rows_kernel(const float* __restrict__ src, int ld_src, int cols, float* __restrict__ dst, int ld_dst,
                                 int64_t rows, int64_t rows_pad) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= rows_pad * ld_dst) return;
  const int64_t r = e / ld_dst;
  const int c = (int)(e % ld_dst);
  dst[e] = (r < rows && c < cols) ? src[r * ld_src + c] : 0.f;
}

__global__ void absmax_kernel(const float* __restrict__ src, int64_t n, int* __restrict__ out_bits) {
  float mx = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    mx = fmaxf(mx, fabsf(src[i]));
  publish_gmax(mx, out_bits);
}

int launch_pack_rows(const float* src, int ld_src, int cols, float* dst, int ld_dst, int64_t rows, int64_t rows_pad,
                     cudaStream_t st) {
  const int64_t n = rows_pad * ld_dst;
  pack_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, ld_src, cols, dst, ld_dst, rows, rows_pad);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int launch_absmax(const float* src, int64_t n, int* out_bits, cudaStream_t st) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > 592) blocks = 592;
  absmax_kernel<<<blocks, 256, 0, st>>>(src, n, out_bits);
  B200_CHECK_LAUNCH();
  return B200_OK;
}


// ---------------------------------------------------------------------------------------------
// Data-parallel optimiser step over NVLink peer memory: reduce-scatter + Adam + all-gather in ONE kernel
// (SURVEY.md §8e).  Replaces  all_reduce(grads || losses)  +  Adam  of the frame-sharded loop.
//
// Every rank owns one contiguous slice of the flat [gradients || 8 losses] buffer.  For its slice it sums the
// W partial buffers (peer loads, fixed rank order: every element is summed exactly once, by one rank, so all ranks
// end with bit-identical parameters), applies Adam (same arithmetic as adam_kernel; the moments of a slice live
// on its owner) and stores the new parameters / the reduced losses into every rank's buffer (peer stores).
// Cross-GPU ordering uses two flag rounds in symmetric memory, numbered by a monotonically increasing epoch:
//   round A  "my partial buffer is complete"  — set at kernel start, awaited by every block before it loads
//   round B  "I have finished reading and writing" — set by the last block of a rank, awaited by that block
//            before the kernel ends, so the next kernel on any rank sees complete parameters and may overwrite
//            its own partial buffer.
// ---------------------------------------------------------------------------------------------
__device__ unsigned int g_dp_ticket = 0u;

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(256) dp_adam_kernel(B200DpComm comm, float* __restrict__ m, float* __restrict__ v,
                                                      int64_t n_params, int64_t n_total, double lr, double b1d,
                                                      double b2d, double epsd, int64_t* __restrict__ step_io,
                                                      unsigned long long* __restrict__ epoch_io) {
  __shared__ float s_step_size, s_bc2_sqrt;
  __shared__ unsigned long long s_epoch;
  const int W = comm.world, R = comm.rank;
  if (threadIdx.x == 0) {
    const double t = (double)(*step_io + 1);
    s_step_size = (float)(lr / (1.0 - pow(b1d, t)));
    s_bc2_sqrt = (float)sqrt(1.0 - pow(b2d, t));
    s_epoch = *epoch_io + 1;
  }
  __syncthreads();
  const unsigned long long epoch = s_epoch;
  // ---- round A: publish "my partials are complete" (once per rank), then wait for every peer
  if (blockIdx.x == 0 && threadIdx.x < W) st_release_sys(comm.flags[threadIdx.x] + R, epoch);
  if (threadIdx.x < W) {
    const unsigned long long* f = comm.flags[R] + threadIdx.x;
    const long long t0 = clock64();
    while (ld_acquire_sys(f) < epoch) {
      if (clock64() - t0 > 20000000000ll) { printf("b200: dp_adam round A timed out (rank %d waits for %d)\n", R, (int)threadIdx.x); __trap(); }
    }
  }
  __syncthreads();
  const float step_size = s_step_size, bc2_sqrt = s_bc2_sqrt;
  const float w1 = (float)(1.0 - b1d), w2 = (float)(1.0 - b2d), b2 = (float)b2d, eps = (float)epsd;
  const int64_t total4 = (n_total + 3) / 4, per = (total4 + W - 1) / W;
  const int64_t begin4 = per * R, end4 = min(total4, per * (R + 1));
  for (int64_t i4 = begin4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i4 < end4; i4 += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = i4 * 4;
    float4 g = *reinterpret_cast<const float4*>(comm.partials[0] + i);
    for (int j = 1; j < W; ++j) {
      const float4 q = *reinterpret_cast<const float4*>(comm.partials[j] + i);
      g.x += q.x; g.y += q.y; g.z += q.z; g.w += q.w;
    }
    float out[4];
    const float ga[4] = {g.x, g.y, g.z, g.w};
    if (i < n_params) {              // parameter block (n_params is a multiple of 4)
      const float4 pp = *reinterpret_cast<const float4*>(comm.params[R] + i);
      float4 mm = *reinterpret_cast<float4*>(m + i), vv = *reinterpret_cast<float4*>(v + i);
      float pa[4] = {pp.x, pp.y, pp.z, pp.w}, ma[4] = {mm.x, mm.y, mm.z, mm.w}, va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        ma[q] = ma[q] + w1 * (ga[q] - ma[q]);
        va[q] = va[q] * b2 + (w2 * ga[q]) * ga[q];
        const float denom = sqrtf(va[q]) / bc2_sqrt + eps;
        out[q] = pa[q] + (-step_size * ma[q]) / denom;
      }
      *reinterpret_cast<float4*>(m + i) = make_float4(ma[0], ma[1], ma[2], ma[3]);
      *reinterpret_cast<float4*>(v + i) = make_float4(va[0], va[1], va[2], va[3]);
      const float4 o = make_float4(out[0], out[1], out[2], out[3]);
      for (int j = 0; j < W; ++j) *reinterpret_cast<float4*>(comm.params[j] + i) = o;
    } else {                          // the loss vector: every rank gets the sums in place
      for (int j = 0; j < W; ++j) *reinterpret_cast<float4*>(const_cast<float*>(comm.partials[j]) + i) = g;
    }
  }
  // ---- round B: the last block of this rank tells every peer "done" and waits for all of them
  __threadfence_system();
  __syncthreads();
  __shared__ bool s_last;
  if (threadIdx.x == 0) s_last = (atomicAdd(&g_dp_ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (s_last) {
    if (threadIdx.x < W) st_release_sys(comm.flags[threadIdx.x] + W + R, epoch);
    if (threadIdx.x < W) {
      const unsigned long long* f = comm.flags[R] + W + threadIdx.x;
      const long long t0 = clock64();
      while (ld_acquire_sys(f) < epoch) {
        if (clock64() - t0 > 20000000000ll) { printf("b200: dp_adam round B timed out (rank %d waits for %d)\n", R, (int)threadIdx.x); __trap(); }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) { *step_io += 1; *epoch_io = epoch; g_dp_ticket = 0u; }
  }
}

int launch_dp_adam(const B200DpComm& comm, float* m, float* v, int64_t n_params, int64_t n_total, double lr,
                   double b1, double b2, double eps, int64_t* step, unsigned long long* epoch, cudaStream_t st) {
  const int64_t total4 = (n_total + 3) / 4, per = (total4 + comm.world - 1) / comm.world;
  int blocks = (int)((per + 255) / 256);
  if (blocks > 132) blocks = 132;                 // all blocks must be co-resident (they wait on remote flags)
  if (blocks < 1) blocks = 1;
  timer_begin(TAG_ADAM, st);
  dp_adam_kernel<<<blocks, 256, 0, st>>>(comm, m, v, n_params, n_total, lr, b1, b2, eps, step, epoch);
  timer_end(TAG_ADAM, st);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

}  // namespace b200
