// Fixed-order sum over a CTA, shared by the float64 reductions that must be bit-identical across calls, CUDA-graph
// replays, batch sizes and ranks (eval_sse.cu, warp_error.cu).
#pragma once

namespace b200 {

// Sum of `v` over a CTA of kThreads threads (a multiple of 32, at most 1024), valid in thread 0; `sh` holds kThreads / 32
// doubles.  Fixed order: xor-shuffle tree in each warp, then warp 0 over the warps.
template <int kThreads>
__device__ __forceinline__ double cta_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < kThreads / 32 ? sh[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  }
  return v;
}

}  // namespace b200
