// Thin inline-PTX layer for the sm_90a kernels: mbarrier, bulk async copy (TMA engine), wgmma (mma / fences) and its
// shared-memory descriptors.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace b200 {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (reported as a CUDA error) instead of a hung GPU.  No call in here (no
// printf): a function call inside a wgmma pipeline makes ptxas serialise every wgmma of the kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000ll) __trap();   // ~2 s at 2 GHz
  }
}

// ------------------------------------------------------------------------------------ thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster; orders the shared-memory operations before it cluster-wide
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the shared::cluster address of the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
// arrive on an mbarrier of another CTA of the cluster (address from mapa_shared).  Default (CTA-scope) release: it
// frees an operand slot whose reads by wgmma have already completed, so no cluster-wide fence is needed.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}

// ------------------------------------------------------------------------------------ bulk copy
// contiguous global -> shared through the TMA engine (UBLKCP), completion on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// the same copy into the same shared-memory offset of every CTA of the cluster in `cta_mask`; each destination CTA's
// mbarrier at the offset of `bar` receives the bytes it got
__device__ __forceinline__ void bulk_g2s_multicast(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar,
                                                   uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------------------------------ wgmma
// A warpgroup (4 consecutive warps, the first a multiple of 4) issues the MMAs together; the accumulator lives in its
// registers: thread (warp w of the group, lane l) holds rows 16w + l/4 and 16w + l/4 + 8, columns 8i + 2(l%4) + {0,1}
// as d[4i + {0,1}] (first row) and d[4i + {2,3}] (second row).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Register budget of a warpgroup (all its threads execute it): producers hand registers to the consumer warpgroups
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// warp index the compiler knows to be warp-uniform (role branches on it are not divergent paths around wgmma)
__device__ __forceinline__ int warp_uniform() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }
// keeps the compiler from moving accumulator accesses across an in-flight wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 256] (+)= A[64 x 16] * B[16 x 256], both operands from shared memory (fp16 in, fp32 accumulate).
// TA / TB: 0 = K-major, 1 = MN-major operand.  scale_d == 0 overwrites D.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[16 x 128], both operands from shared memory (fp16 in, fp32 accumulate).
// TA / TB: 0 = K-major, 1 = MN-major operand.  scale_d == 0 overwrites D.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

// D[64 x 64] (+)= A[64 x 16] * B[16 x 64], both operands from shared memory (fp16 in, fp32 accumulate).
// TA / TB: 0 = K-major, 1 = MN-major operand.  scale_d == 0 overwrites D.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

// D[64 x 8] (+)= A[64 x 16] * B[16 x 8], both operands from shared memory (fp16 in, fp32 accumulate).
// TA / TB: 0 = K-major, 1 = MN-major operand.  scale_d == 0 overwrites D.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_n8(float (&d)[4], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, %7, %8;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TA), "n"(TB)
      : "memory");
}

// ------------------------------------------------------------------------------------ descriptors
// wgmma shared-memory matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout type [62,64)
// (1 = 128-byte swizzle).  K-major SW128: SBO = stride of 8-row groups (LBO unused); MN-major SW128: LBO = stride of
// 64-element MN blocks, SBO = stride of 8-deep K groups.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// K-major 64-byte swizzle (layout type 2): rows of 64 B (32 fp16 k), 16-byte chunk index XOR-ed with (row / 2) % 4,
// SBO = stride of 8-row groups (512 B when dense); LBO unused
__device__ __forceinline__ uint64_t make_desc_sw64(uint32_t smem_addr, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)2 << 62;
  return d;
}
// no swizzle (layout type 0), for an operand of 8-element (16-byte) rows: MN-major, 8 MN elements x 8 k = one 128-byte
// core matrix, k groups of 8 at consecutive 128 bytes.  With N = 8 there is one MN group, so LBO and SBO (whose roles
// the interleaved MN-major layout swaps against the swizzled ones) are both the 128-byte k-group stride.
__device__ __forceinline__ uint64_t make_desc_rows16(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)(128 >> 4) << 16;
  d |= (uint64_t)(128 >> 4) << 32;
  return d;
}

// ------------------------------------------------------------------------------------ fp16 split
// v -> (hi, lo) with hi = rn_f16(v), lo = rn_f16(v - hi); saturating (no inf).  v must already be scaled.
__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
  unsigned short h, l;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(v));
  const float hf = __half2float(__ushort_as_half(h));
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(l) : "f"(v - hf));
  hi = __ushort_as_half(h);
  lo = __ushort_as_half(l);
}
__device__ __forceinline__ uint32_t pack2(__half a, __half b) {   // a -> low 16 bits (even k)
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

}  // namespace ptx
}  // namespace b200

namespace b200 {
namespace ptx {
// contiguous shared -> global through the TMA engine, tracked by bulk async-groups
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// two floats -> packed half2 (a -> low half), round to nearest, saturating
__device__ __forceinline__ uint32_t cvt_pack_f16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// split two already-scaled floats into packed (hi, lo) half2 words
__device__ __forceinline__ void split2_f16(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = cvt_pack_f16x2(a, b);
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = cvt_pack_f16x2(a - hf.x, b - hf.y);
}
}  // namespace ptx
}  // namespace b200

namespace b200 {
namespace ptx {
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
}  // namespace ptx
}  // namespace b200

namespace b200 {
namespace ptx {
// ---- pairs of fp32 values in one 64-bit word, operated on lane by lane (each op rounds exactly like its scalar form)
__device__ __forceinline__ uint64_t pack2f(float a, float b) { uint64_t r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ uint64_t pack2u(uint32_t a, uint32_t b) { uint64_t r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ void unpack2f(uint64_t v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1; unpack2f(a, a0, a1); unpack2f(b, b0, b1); unpack2f(c, c0, c1);
  return pack2f(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1; unpack2f(a, a0, a1); unpack2f(b, b0, b1);
  return pack2f(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t sub2(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1; unpack2f(a, a0, a1); unpack2f(b, b0, b1);
  return pack2f(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
// 2-term fp16 split of two already-scaled floats: same values as split2_f16
__device__ __forceinline__ void split2_packed(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = cvt_pack_f16x2(a, b);
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  float d0, d1;
  unpack2f(sub2(pack2f(a, b), pack2f(hf.x, hf.y)), d0, d1);
  lo = cvt_pack_f16x2(d0, d1);
}
// appends the ReLU flag of v (v >= +0: the output of fmaxf(z, 0)) to a bit string: flag = v > 0 <=> 0 - bits(v) is
// negative.  After n appends the FIRST value's flag is bit n-1.
__device__ __forceinline__ uint32_t push_flag(uint32_t bw, float v) {
  return __funnelshift_l((uint32_t)(-(int)__float_as_uint(v)), bw, 1);
}
}  // namespace ptx
}  // namespace b200
