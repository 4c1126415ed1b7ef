// Thin inline-PTX wrappers for the sm_90a features the UniVTG hot path uses:
// mbarrier, TMA (cp.async.bulk.tensor, cluster multicast), wgmma fences and the GMMA shared-memory descriptor.
// sm_90a only - no other arch is supported.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace uv {

#define UV_DEVINL __device__ __forceinline__

UV_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

UV_DEVINL uint32_t lane_id() { return threadIdx.x & 31; }

UV_DEVINL bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// programmatic dependent launch (see launch_k, kernels.h).  No-ops when the kernel was launched without the attribute.
// ----------------------------------------------------------------------------------------------
UV_DEVINL void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
UV_DEVINL void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// first statement of every kernel: let the next grid get scheduled, then wait until everything before this grid is visible
UV_DEVINL void pdl_prologue() {
  pdl_launch_dependents();
  pdl_wait();
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
UV_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
UV_DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
UV_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

UV_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
UV_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
UV_DEVINL bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
UV_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
UV_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load, coordinates (c0 = innermost element index, c1 = row index)
UV_DEVINL void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
UV_DEVINL uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
UV_DEVINL void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `smem_addr` (a shared::cta address of this CTA) in CTA `rank` of the cluster
UV_DEVINL uint32_t mapa_shared(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
// arrive on an mbarrier that lives in another CTA of the cluster (address from mapa_shared)
UV_DEVINL void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// 2-D tiled load multicast to every CTA of `cta_mask`: the tile lands at the same smem offset in each of them and the bytes are
// credited to the mbarrier at the same offset in each of them.
UV_DEVINL void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
UV_DEVINL void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, sm_90a): fences and the shared-memory matrix descriptor.  The MMAs themselves are in wgmma.cuh.
// ----------------------------------------------------------------------------------------------
UV_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
UV_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
UV_DEVINL void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across a wgmma that is still in flight
UV_DEVINL void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }
UV_DEVINL void reg_fence(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }
template <uint32_t kRegs>
UV_DEVINL void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs));
}
template <uint32_t kRegs>
UV_DEVINL void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs));
}
// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
UV_DEVINL void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// Shared-memory matrix descriptor for a SWIZZLE_128B tile of 16-bit elements (sm_90 GMMA encoding).
//   K-major : rows of 128 B (64 elements of K), 8-row swizzle atoms of 1024 B stacked along M/N.
//             SBO = 1024 B (next 8-row group); LBO unused (1).  One k-step of 16 elements = +32 B.
//   MN-major: "rows" of 128 B are 64 consecutive M/N elements for one k; 8 k's form a 1024 B atom.
//             SBO = 1024 B (next 8 k's); LBO = byte distance between 64-element M/N blocks.  One k-step = +2048 B.
// bits [0,14) addr>>4, [16,30) LBO>>4, [32,46) SBO>>4, [62,64) layout = 1 (128B swizzle).
UV_DEVINL uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// ----------------------------------------------------------------------------------------------
// small math helpers
// ----------------------------------------------------------------------------------------------
UV_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// 32-byte global accesses (one whole sector per thread) as two 128-bit accesses.  Addresses must be 32-byte aligned.
UV_DEVINL void st_global_256(void* p, const uint32_t (&w)[8]) {
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = make_uint4(w[0], w[1], w[2], w[3]);
  q[1] = make_uint4(w[4], w[5], w[6], w[7]);
}
UV_DEVINL void st_global_256f(float* p, float a0, float a1, float a2, float a3, float a4, float a5, float a6, float a7) {
  float4* q = reinterpret_cast<float4*>(p);
  q[0] = make_float4(a0, a1, a2, a3);
  q[1] = make_float4(a4, a5, a6, a7);
}
UV_DEVINL void ld_global_256f(const float* p, float* v) {
  const float4 a = reinterpret_cast<const float4*>(p)[0];
  const float4 b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
// one 128-bit reduction (four fp32 adds, relaxed, gpu scope) - addr must be 16-byte aligned
UV_DEVINL void red_add_f32x4(float* addr, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// one halving step of warp_colsum16.  OFF is a template parameter so that every index into v is a compile-time constant: with
// a loop over OFF the compiler left the inner loop rolled in the GEMM's FULL epilogue, and the dynamic index put v (and with it
// every value of the epilogue) in local memory.
template <int OFF>
UV_DEVINL void colsum16_step(float (&v)[16], int lane) {
  const bool hi = (lane & OFF) != 0;
#pragma unroll
  for (int k = 0; k < OFF; ++k) {
    const float send = hi ? v[k] : v[k + OFF];
    const float keep = hi ? v[k + OFF] : v[k];
    v[k] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
  }
}
// Transposing reduction of 16 values per lane across the warp (16 shuffles instead of 16 x 5): on return every lane l holds
// the sum over all 32 lanes of their v[l & 15] (v is clobbered).
UV_DEVINL float warp_colsum16(float (&v)[16], int lane) {
  colsum16_step<8>(v, lane);
  colsum16_step<4>(v, lane);
  colsum16_step<2>(v, lane);
  colsum16_step<1>(v, lane);
  return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 16);
}
UV_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// erf via Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7): ~4x fewer instructions than erff in the GEMM epilogue.
UV_DEVINL float erf_fast(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  float y = fmaf(1.061405429f, t, -1.453152027f);
  y = fmaf(y, t, 1.421413741f);
  y = fmaf(y, t, -0.284496736f);
  y = fmaf(y, t, 0.254829592f);
  y = y * t;
  const float r = fmaf(-y, __expf(-ax * ax), 1.0f);
  return copysignf(r, x);
}
// gelu(x) = 0.5 x (1 + erf(x / sqrt 2)) = 0.5 (x + |x| erf(|x| / sqrt 2)), with the same A&S 7.1.26 erf, constants folded
UV_DEVINL float gelu_erf(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f * 0.70710678118654752440f, ax, 1.0f));
  float y = fmaf(1.061405429f, t, -1.453152027f);
  y = fmaf(y, t, 1.421413741f);
  y = fmaf(y, t, -0.284496736f);
  y = fmaf(y, t, 0.254829592f);
  y = y * t;
  const float e = exp2f(ax * ax * (-0.5f * 1.4426950408889634f));  // exp(-x^2 / 2)
  const float r = fmaf(-y, e, 1.0f);                                // erf(|x| / sqrt 2)
  return 0.5f * fmaf(ax, r, x);
}
// d/dx gelu(x) = Phi(x) + x phi(x), Phi(x) = 0.5 (1 + erf(x / sqrt 2)), phi(x) = exp(-x^2/2) / sqrt(2 pi); same erf as above
UV_DEVINL float gelu_erf_grad(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f * 0.70710678118654752440f, ax, 1.0f));
  float y = fmaf(1.061405429f, t, -1.453152027f);
  y = fmaf(y, t, 1.421413741f);
  y = fmaf(y, t, -0.284496736f);
  y = fmaf(y, t, 0.254829592f);
  y = y * t;
  const float e = exp2f(ax * ax * (-0.5f * 1.4426950408889634f));
  const float r = fmaf(-y, e, 1.0f);  // erf(|x| / sqrt 2)
  return fmaf(0.5f, copysignf(r, x), 0.5f) + x * 0.3989422804014327f * e;
}
// gelu(x) and d/dx gelu(x) together (they share the reciprocal, the polynomial and the exponential)
UV_DEVINL void gelu_erf_both(float x, float& g, float& dg) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f * 0.70710678118654752440f, ax, 1.0f));
  float y = fmaf(1.061405429f, t, -1.453152027f);
  y = fmaf(y, t, 1.421413741f);
  y = fmaf(y, t, -0.284496736f);
  y = fmaf(y, t, 0.254829592f);
  y = y * t;
  const float e = exp2f(ax * ax * (-0.5f * 1.4426950408889634f));  // exp(-x^2 / 2)
  const float r = fmaf(-y, e, 1.0f);                                // erf(|x| / sqrt 2)
  g = 0.5f * fmaf(ax, r, x);
  dg = fmaf(0.5f, copysignf(r, x), 0.5f) + x * 0.3989422804014327f * e;
}
UV_DEVINL bool pos16(uint16_t h) { return (h & 0x8000u) == 0 && (h & 0x7fffu) != 0; }  // 16-bit float > 0 (fp16 or bf16)

// 16-bit MMA operand storage.  fmt: 0 = fp16 (default; 11-bit significand), 1 = bf16 (8-bit).
// The format is a run-time property of a plan (it only changes conversions + the instruction descriptor).
UV_DEVINL uint16_t cvt16(float v, int fmt) {
  return fmt ? __bfloat16_as_ushort(__float2bfloat16_rn(v)) : __half_as_ushort(__float2half_rn(v));
}
UV_DEVINL uint32_t cvt16x2(float lo, float hi, int fmt) {
  return (uint32_t)cvt16(lo, fmt) | ((uint32_t)cvt16(hi, fmt) << 16);
}
UV_DEVINL float ld16(uint16_t v, int fmt) {
  return fmt ? __bfloat162float(__ushort_as_bfloat16(v)) : __half2float(__ushort_as_half(v));
}
// Split fp16 ("fp16x3", operand_format 2): a value v is stored as two fp16 planes, hi = fp16(v) (cvt16 with fmt 0) and
// lo = fp16(v - hi).  v - hi is exact in fp32, and hi + lo is exact in fp32 again.
UV_DEVINL uint16_t cvt16_lo(float v) { return cvt16(v - ld16(cvt16(v, 0), 0), 0); }
UV_DEVINL uint32_t cvt16x2_lo(float a, float b) { return (uint32_t)cvt16_lo(a) | ((uint32_t)cvt16_lo(b) << 16); }
UV_DEVINL float ld16x3(uint16_t hi, uint16_t lo) { return ld16(hi, 0) + ld16(lo, 0); }

}  // namespace uv
