// fp32 CUDA-core path of the IMLP layers (B200_PREC_FP32): a register-blocked SGEMM with fused
// epilogues, driven layer by layer.  This is the bit-faithful-fp32 mode (FFMA, fp32 accumulate) used
// for strict parity and as the on-device cross-check of the tensor-core path (mlp_tc.cu).
//
// Restates: nn.Linear stack + ReLU + skip concat + tanh of
//   src/models/stage_1/implicit_neural_networks.py:62-81 and its autograd.
#include "common.cuh"

namespace b200 {

// C[i][j] (op)= epilogue( sum_r P(i,r) * Q(r,j) )
//   P_RC: P(i,r) = P[i*ldp + r]   (r contiguous)   else P[r*ldp + i]   (i contiguous)
//   Q_RC: Q(r,j) = Q[j*ldq + r]   (r contiguous)   else Q[r*ldq + j]   (j contiguous)
struct GemmArgs {
  const float* P; int64_t ldp;
  const float* Q; int64_t ldq;
  float* C; int64_t ldc;
  int I, J, R;
  const float* bias;        // per j, added before the activation (may be null)
  int act;                  // 0 none, 1 relu, 2 tanh
  const float* mask; int64_t ld_mask;   // multiply by (mask[i][j] > 0) when non-null
  int atomic;               // accumulate with atomicAdd (split-R) instead of storing
  float* bias_grad;         // wgrad only: bias_grad[i] += sum_r P(i,r)
  // row validity (RowSpan).  rows_on_i: the I dimension indexes batch rows (fwd/dgrad),
  // otherwise the R dimension does (wgrad, split over blockIdx.z in chunks of r_chunk).
  int rows_on_i;
  int64_t cap; const int* n_valid;
  int r_chunk;
  int tag;                  // KernelTag timed by b200_set_kernel_timer (0: none)
  float scale;              // multiplies the accumulator first (0 -> 1)
};

constexpr int BI = 128, BJ = 128, BR = 16, PADW = 132, GEMM_THREADS = 256;

template <bool RC>
__device__ __forceinline__ void load_tile(float (*S)[PADW], const float* __restrict__ M, int64_t ld,
                                          int o0, int O, int r0, int r_end, int tid) {
  // fills S[r][o] for r in [0,BR), o in [0,128) with M(o0+o, r0+r) (0 outside bounds)
  const bool vec = ((ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(M) & 15) == 0);
  if (RC) {
    // element (o, r) at M[(o0+o)*ld + r0 + r]: 4 consecutive r per thread
#pragma unroll
    for (int it = 0; it < (BI * BR / 4) / GEMM_THREADS; ++it) {
      const int e = tid + it * GEMM_THREADS;
      const int o = e / (BR / 4), r4 = (e % (BR / 4)) * 4;
      const int go = o0 + o, gr = r0 + r4;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (go < O) {
        const float* src = M + (int64_t)go * ld + gr;
        if (vec && ((r0 & 3) == 0) && gr + 3 < r_end) {
          const float4 t = *reinterpret_cast<const float4*>(src);
          v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) if (gr + q < r_end) v[q] = src[q];
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) S[r4 + q][o] = v[q];
    }
  } else {
    // element (o, r) at M[(r0+r)*ld + o0 + o]: 4 consecutive o per thread
#pragma unroll
    for (int it = 0; it < (BI * BR / 4) / GEMM_THREADS; ++it) {
      const int e = tid + it * GEMM_THREADS;
      const int r = e / (BI / 4), o4 = (e % (BI / 4)) * 4;
      const int gr = r0 + r, go = o0 + o4;
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gr < r_end) {
        const float* src = M + (int64_t)gr * ld + go;
        if (vec && ((o0 & 3) == 0) && go + 3 < O) {
          t = *reinterpret_cast<const float4*>(src);
        } else {
          if (go + 0 < O) t.x = src[0];
          if (go + 1 < O) t.y = src[1];
          if (go + 2 < O) t.z = src[2];
          if (go + 3 < O) t.w = src[3];
        }
      }
      *reinterpret_cast<float4*>(&S[r][o4]) = t;
    }
  }
}

template <bool P_RC, bool Q_RC>
__global__ void __launch_bounds__(GEMM_THREADS, 2) sgemm_kernel(GemmArgs a) {
  __shared__ __align__(16) float Ps[2][BR][PADW];
  __shared__ __align__(16) float Qs[2][BR][PADW];
  const int tid = threadIdx.x;
  const int i0 = blockIdx.x * BI, j0 = blockIdx.y * BJ;
  int r_begin = 0, r_end = a.R;
  if (a.rows_on_i) {
    if (a.n_valid && a.cap > 0 && (i0 % a.cap) >= *a.n_valid) return;   // tile of padding rows only
  } else {
    // split over the batch rows: blockIdx.z = group * chunks_per_group + chunk, so that no chunk
    // straddles two row groups; clamp to the whole 128-row tiles the forward pass touched
    const int64_t cap = a.cap > 0 ? a.cap : (int64_t)a.R;
    const int cpg = (int)((cap + a.r_chunk - 1) / a.r_chunk);
    const int64_t gbase = (int64_t)(blockIdx.z / cpg) * cap;
    int64_t valid = cap;
    if (a.n_valid && a.cap > 0)
      valid = min(cap, (int64_t)((*a.n_valid + kTileRows - 1) / kTileRows) * kTileRows);
    const int64_t rb = gbase + (int64_t)(blockIdx.z % cpg) * a.r_chunk;
    r_begin = (int)rb;
    r_end = (int)min(min(gbase + valid, rb + a.r_chunk), (int64_t)a.R);
    if (r_begin >= r_end) return;
  }
  const int ty = tid / 16, tx = tid % 16;
  float acc[8][8];
#pragma unroll
  for (int u = 0; u < 8; ++u)
#pragma unroll
    for (int v = 0; v < 8; ++v) acc[u][v] = 0.f;
  float bsum[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) bsum[u] = 0.f;
  const bool do_bsum = (a.bias_grad != nullptr) && blockIdx.y == 0 && tx == 0;

  int buf = 0;
  load_tile<P_RC>(Ps[0], a.P, a.ldp, i0, a.I, r_begin, r_end, tid);
  load_tile<Q_RC>(Qs[0], a.Q, a.ldq, j0, a.J, r_begin, r_end, tid);
  __syncthreads();
  for (int r0 = r_begin; r0 < r_end; r0 += BR) {
    if (r0 + BR < r_end) {
      load_tile<P_RC>(Ps[buf ^ 1], a.P, a.ldp, i0, a.I, r0 + BR, r_end, tid);
      load_tile<Q_RC>(Qs[buf ^ 1], a.Q, a.ldq, j0, a.J, r0 + BR, r_end, tid);
    }
#pragma unroll
    for (int r = 0; r < BR; ++r) {
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
      if (do_bsum) {
#pragma unroll
        for (int u = 0; u < 8; ++u) bsum[u] += p[u];
      }
    }
    __syncthreads();
    buf ^= 1;
  }
  // epilogue
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int i = i0 + ty * 8 + u;
    if (i >= a.I) continue;
#pragma unroll
    for (int v = 0; v < 8; ++v) {
      const int j = j0 + tx * 8 + v;
      if (j >= a.J) continue;
      float val = a.scale != 0.f ? acc[u][v] * a.scale : acc[u][v];
      if (a.bias) val += a.bias[j];
      if (a.act == 1) val = fmaxf(val, 0.f);
      else if (a.act == 2) val = tanhf(val);
      if (a.mask) val = (a.mask[(int64_t)i * a.ld_mask + j] > 0.f) ? val : 0.f;
      float* dst = a.C + (int64_t)i * a.ldc + j;
      if (a.atomic) atomicAdd(dst, val); else *dst = val;
    }
  }
  if (do_bsum) {
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int i = i0 + ty * 8 + u;
      if (i < a.I) atomicAdd(a.bias_grad + i, bsum[u]);
    }
  }
}

static int launch_gemm(const GemmArgs& a, bool p_rc, bool q_rc, cudaStream_t st) {
  dim3 grid((a.I + BI - 1) / BI, (a.J + BJ - 1) / BJ, 1);
  if (!a.rows_on_i) {
    const int64_t cap = a.cap > 0 ? a.cap : (int64_t)a.R;
    grid.z = (unsigned)(((int64_t)a.R + cap - 1) / cap * ((cap + a.r_chunk - 1) / a.r_chunk));
  }
  timer_begin(a.tag, st);
  if (p_rc && q_rc) sgemm_kernel<true, true><<<grid, GEMM_THREADS, 0, st>>>(a);
  else if (p_rc && !q_rc) sgemm_kernel<true, false><<<grid, GEMM_THREADS, 0, st>>>(a);
  else if (!p_rc && !q_rc) sgemm_kernel<false, false><<<grid, GEMM_THREADS, 0, st>>>(a);
  else { set_error("unsupported gemm layout"); return B200_ERR_INVALID; }
  timer_end(a.tag, st);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int simt_gemm_nn_scaled(const float* A, const float* B, float* C, int M, int N, int K, float scale, cudaStream_t st) {
  GemmArgs g{};
  g.P = A; g.ldp = M;          // P(i, r) = A[r*M + i]   (i contiguous)
  g.Q = B; g.ldq = N;          // Q(r, j) = B[r*N + j]   (j contiguous)
  g.C = C; g.ldc = N; g.I = M; g.J = N; g.R = K; g.rows_on_i = 1; g.scale = scale;
  return launch_gemm(g, false, false, st);
}

// dz[i][j] = dy[i][j] * (1 - y[i][j]^2)   (tanh backward), or a copy when tanh is off
__global__ void out_grad_kernel(const float* __restrict__ dy, const float* __restrict__ y,
                                float* __restrict__ dz, int64_t n, int use_tanh) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float g = dy[i];
  if (use_tanh) { const float t = y[i]; dz[i] = g * (1.f - t * t); }
  else dz[i] = g;
}

int simt_mlp_forward(const MlpShape& s, const float* params, const float* x, int ldx, const RowSpan& span,
                     const MlpScratch& sc, float* y, cudaStream_t st) {
  for (int l = 0; l < s.L; ++l) {
    GemmArgs a{};
    if (l == 0 && s.pe == 0) { a.P = x; a.ldp = ldx; }
    else { a.P = sc.act[l]; a.ldp = s.K[l]; }
    a.Q = params + s.w_off[l]; a.ldq = s.K[l];
    a.I = (int)span.rows; a.J = s.N[l]; a.R = s.K[l];
    a.bias = params + s.b_off[l];
    a.rows_on_i = 1; a.cap = span.cap; a.n_valid = span.n_valid;
    if (l == s.L - 1) { a.C = y; a.ldc = s.out_dim; a.act = s.tanh_out ? 2 : 0; }
    else { a.C = sc.act[l + 1]; a.ldc = s.K[l + 1]; a.act = 1; }
    if (l == 1) a.tag = s.pe == 0 ? TAG_MAP_FWD : TAG_ATLAS_FWD;      // one 256x256 hidden layer
    B200_PROPAGATE(launch_gemm(a, true, true, st));
  }
  return B200_OK;
}

int simt_mlp_backward(const MlpShape& s, const float* params, const float* x, int ldx, const RowSpan& span,
                      const MlpScratch& sc, const float* dy, float* dparams, float* d_in, int ld_din,
                      cudaStream_t st) {
  const int64_t n_out = span.rows * s.out_dim;
  int cur = 0;
  out_grad_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, st>>>(dy, sc.y, sc.dz[cur], n_out, s.tanh_out ? 1 : 0);
  B200_CHECK_LAUNCH();
  for (int l = s.L - 1; l >= 0; --l) {
    const float* A = (l == 0 && s.pe == 0) ? x : sc.act[l];
    const int64_t lda = (l == 0 && s.pe == 0) ? ldx : s.K[l];
    const int ldz = s.N[l];
    // weight + bias gradient: dW[n][k] += sum_m dZ[m][n] * A[m][k]
    GemmArgs w{};
    w.P = sc.dz[cur]; w.ldp = ldz;       // P(i=n, r=m) = dZ[m*ldz + n]  (i contiguous)
    w.Q = A; w.ldq = lda;                // Q(r=m, j=k) = A[m*lda + k]   (j contiguous)
    w.C = dparams + s.w_off[l]; w.ldc = s.K[l];
    w.I = s.N[l]; w.J = s.K[l]; w.R = (int)span.rows;
    w.atomic = 1; w.bias_grad = dparams + s.b_off[l];
    w.rows_on_i = 0; w.cap = span.cap; w.n_valid = span.n_valid;
    w.r_chunk = 1024;
    if (l == 1 && s.pe == 0) w.tag = TAG_WGRAD;
    B200_PROPAGATE(launch_gemm(w, false, false, st));
    // input gradient
    if (l > 0 || d_in != nullptr) {
      GemmArgs g{};
      g.P = sc.dz[cur]; g.ldp = ldz;                       // P(i=m, r=n)
      g.Q = params + s.w_off[l]; g.ldq = s.K[l];           // Q(r=n, j=k) = W[n*K + k]
      g.I = (int)span.rows; g.R = s.N[l];
      g.rows_on_i = 1; g.cap = span.cap; g.n_valid = span.n_valid;
      if (l > 0) {
        g.J = s.hidden;                                    // skip columns are detached: no gradient
        g.C = sc.dz[cur ^ 1]; g.ldc = s.hidden;
        g.mask = sc.act[l]; g.ld_mask = s.K[l];            // ReLU'(h) from the stored post-ReLU value
        if (l == 2) g.tag = s.pe == 0 ? TAG_MAP_BWD : TAG_ATLAS_BWD;
      } else {
        g.J = s.K[0]; g.C = d_in; g.ldc = ld_din;
      }
      B200_PROPAGATE(launch_gemm(g, true, false, st));
      cur ^= 1;
    }
  }
  return B200_OK;
}

}  // namespace b200
