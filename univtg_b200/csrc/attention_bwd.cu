// Attention backward on wgmma (SURVEY.md A.6): per (batch, head, 128-key tile) CTA, loop over 128-query tiles, each processed
// as two 64-query halves.  Everything is computed transposed (rows = keys), so that P^T and dS^T come out of the accumulators
// in the layout of a wgmma A fragment and the dV / dK products take them straight from registers:
//   S^T  = K Q^T   (recomputed)                      P^T  = exp(scale * S^T - lse)  (key padding -> 0)
//   dP^T = V dO^T                                    dS^T = P^T o (dP^T - delta) * scale
//   dV  += P^T dO       dK += dS^T Q                 dQ_i = dS K  (dS^T staged through smem; fp32 global accumulation over key tiles)
// Two warpgroups, warpgroup w owns keys [64 w, 64 w + 64) of the tile (S^T / dP^T: wgmma m64n64, A = K / V rows, B = Q / dO
// rows, all K-major; dV / dK: A from registers, B = dO / Q rows of the half, MN-major).  dQ of a half: A = dS^T (MN-major smem,
// M = queries), B = K (MN-major, N = dh); with dh = 128 each warpgroup computes 64 of the dh columns, with dh = 64 warpgroup 0.
// Q, K, V, dO, P and dS share one 16-bit format (a wgmma takes A and B in one format).
#include <math.h>

#include "backward.h"
#include "kernels.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace uv {

template <int DH>
struct AttnBwdCfg {
  static constexpr int kTile = 128 * DH * 2;  // Q, dO, K, V tiles: DH/64 boxes of [128 rows x 64]
  static constexpr int kDS = 128 * 128;       // dS^T of one 64-query half: [128 keys x 64 queries] 16-bit, 128B-swizzled rows
  static constexpr int kSmemBytes = 1024 + 4 * kTile + kDS + 3 * 128 * 4 + 64;
};

// DROP = 1: the forward's attention dropout M is regenerated (attn_drop_block) and applied as dV += (P o M)^T dO and
// dS^T = P^T o (M o dP^T - delta).  delta = rowsum(dO o O) needs no change: O is the dropped output.
template <int DH, int BF, int DROP>
__global__ void __launch_bounds__(256, 1) attention_bwd_wgmma_kernel(const __grid_constant__ AttnBwdArgs a) {
  using Cfg = AttnBwdCfg<DH>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sdO = sQ + Cfg::kTile;
  uint8_t* sK = sdO + Cfg::kTile;
  uint8_t* sV = sK + Cfg::kTile;
  uint8_t* sdS = sV + Cfg::kTile;
  float* s_kbias = reinterpret_cast<float*>(sdS + Cfg::kDS);  // [128] 0 / -inf per key of this CTA's key tile
  float* s_lse2 = s_kbias + 128;                              // [128] lse * log2(e) per query of the tile (+inf: no query)
  float* s_dlt = s_lse2 + 128;                                // [128] delta per query of the tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_dlt + 128);
  uint64_t* kv_full = bars + 0;
  uint64_t* qdo_full = bars + 1;

  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int tid = threadIdx.x & 127;
  const int fr = 16 * (tid >> 5) + (lane >> 2);  // accumulator rows fr, fr + 8; columns 8 i + fc, + 1
  const int fc = 2 * (lane & 3);
  const int j = blockIdx.x;  // key tile
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int L = a.L;
  const int num_q = (L + 127) / 128;
  const size_t ld3 = (size_t)3 * a.d;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&a.tm_qkv);
    tma_prefetch_desc(&a.tm_do);
    mbar_init(kv_full, 1);
    mbar_init(qdo_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // setup done; everything below reads the previous kernels' outputs
  const DropSpec drop = drop_resolve(a.drop);  // (the seed is read after the PDL wait: a preceding kernel may write it)
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(kv_full, 2 * Cfg::kTile);
#pragma unroll
    for (int kb = 0; kb < DH / 64; ++kb) {
      tma_load_2d(sK + kb * 16384, &a.tm_qkv, kv_full, a.d + h * DH + kb * 64, b * L + j * 128);
      tma_load_2d(sV + kb * 16384, &a.tm_qkv, kv_full, 2 * a.d + h * DH + kb * 64, b * L + j * 128);
    }
  }
  if (threadIdx.x < 128) {
    const int key = j * 128 + threadIdx.x;
    s_kbias[threadIdx.x] = (key < L && a.key_mask[(size_t)b * L + key] != 0.f) ? 0.f : -INFINITY;
  }
  const float c_log2e = 1.4426950408889634f;
  const float sc2 = a.scale * c_log2e;
  const uint32_t uQ = smem_u32(sQ), udO = smem_u32(sdO), uK = smem_u32(sK), uV = smem_u32(sV), udS = smem_u32(sdS);

  float dv[DH / 2], dk[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) dv[i] = dk[i] = 0.f;

  for (int i = 0; i < num_q; ++i) {
    __syncthreads();  // every wgmma of the previous query tile has retired: Q / dO tiles and the per-query rows are free
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(qdo_full, 2 * Cfg::kTile);
#pragma unroll
      for (int kb = 0; kb < DH / 64; ++kb) {
        tma_load_2d(sQ + kb * 16384, &a.tm_qkv, qdo_full, h * DH + kb * 64, b * L + i * 128);
        tma_load_2d(sdO + kb * 16384, &a.tm_do, qdo_full, h * DH + kb * 64, b * L + i * 128);
      }
    }
    if (threadIdx.x < 128) {
      const int qi = i * 128 + threadIdx.x;
      const bool qvalid = qi < L;
      s_lse2[threadIdx.x] = qvalid ? a.lse[((size_t)b * a.H + h) * L + qi] * c_log2e : INFINITY;
      s_dlt[threadIdx.x] = qvalid ? a.delta[((size_t)b * a.H + h) * L + qi] : 0.f;
    }
    __syncthreads();
    if (i == 0) mbar_wait(kv_full, 0);
    mbar_wait(qdo_full, i & 1);

#pragma unroll 1
    for (int hq = 0; hq < 2; ++hq) {
      // keep-bits of this thread's 32 elements of the half, packed before the accumulators are live: element (block c, key row
      // fr + 8 r, query column 8 c + fc + e) -> bit 4 c + 2 r + e.  Call (c >> 1, e) covers queries {i0, i0 + 8} x keys
      // {j0, j0 + 1, j0 + 8, j0 + 9}; this thread's keys differ in bit 3 (r) and share bit 0, so it uses 4 of the 8 lanes.
      uint32_t mb = 0u;
      if constexpr (DROP != 0) {
        const unsigned int bh = (unsigned int)(b * a.H + h), key0 = (unsigned int)(j * 128 + wg * 64 + fr);
        const unsigned int half = key0 & 1u;
#pragma unroll
        for (int cp = 0; cp < 4; ++cp) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const uint4 rr = attn_drop_block(drop, bh, (unsigned int)(i * 128 + hq * 64 + 16 * cp + fc + e), key0 & ~9u);
            const uint32_t w[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
            for (int cq = 0; cq < 2; ++cq)
#pragma unroll
              for (int r = 0; r < 2; ++r) {  // word 2 (query bit 3 = cq) + (key bit 3 = r), lane half = key bit 0
                const uint32_t v = half ? (w[2 * cq + r] >> 16) : (w[2 * cq + r] & 0xffffu);
                mb |= (v >= drop.thresh ? 1u : 0u) << (4 * (2 * cp + cq) + 2 * r + e);
              }
          }
        }
      }
      float st[32], dpt[32];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < DH / 16; ++ks) {
        const uint32_t off = (ks / 4) * 16384 + (ks % 4) * 32;
        WG<64, BF>::template ss<0, 0>(st, make_smem_desc_sw128(uK + wg * 8192 + off, 16, 1024),
                                      make_smem_desc_sw128(uQ + hq * 8192 + off, 16, 1024), ks > 0 ? 1u : 0u);
      }
#pragma unroll
      for (int ks = 0; ks < DH / 16; ++ks) {
        const uint32_t off = (ks / 4) * 16384 + (ks % 4) * 32;
        WG<64, BF>::template ss<0, 0>(dpt, make_smem_desc_sw128(uV + wg * 8192 + off, 16, 1024),
                                      make_smem_desc_sw128(udO + hq * 8192 + off, 16, 1024), ks > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        reg_fence(st[e]);
        reg_fence(dpt[e]);
      }
      // P^T and dS^T (rows = keys fr / fr + 8 of this warpgroup, columns = queries 64 hq + 8 c + fc + {0, 1})
      const float kb2[2] = {s_kbias[wg * 64 + fr], s_kbias[wg * 64 + fr + 8]};
      uint32_t pf[4][4], df[4][4];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float p[2], d[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = hq * 64 + 8 * c + fc + e;
            p[e] = exp2f(st[4 * c + 2 * r + e] * sc2 + kb2[r] - s_lse2[col]);
            if constexpr (DROP != 0) {
              const bool keep = (mb >> (4 * c + 2 * r + e)) & 1u;
              d[e] = p[e] == 0.f ? 0.f : p[e] * ((keep ? dpt[4 * c + 2 * r + e] * drop.scale : 0.f) - s_dlt[col]) * a.scale;
              p[e] = keep ? p[e] * drop.scale : 0.f;  // P o M feeds the dV product
            } else {
              d[e] = p[e] == 0.f ? 0.f : p[e] * (dpt[4 * c + 2 * r + e] - s_dlt[col]) * a.scale;
            }
          }
          // accumulator block c, row half r -> A-fragment k-chunk c / 2, register (c & 1) * 2 + r
          pf[c >> 1][(c & 1) * 2 + r] = cvt16x2(p[0], p[1], BF);
          df[c >> 1][(c & 1) * 2 + r] = cvt16x2(d[0], d[1], BF);
          // dS^T row -> smem: 128 B per key row (64 queries), 16-byte chunk c XOR-swizzled with row % 8
          const int row = wg * 64 + fr + 8 * r;
          *reinterpret_cast<uint32_t*>(sdS + row * 128 + ((c ^ (row & 7)) << 4) + fc * 2) = df[c >> 1][(c & 1) * 2 + r];
        }
      }
      fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < 4; ++kc)  // contraction over the 64 queries of the half, 16 per step = two 1024 B atoms
        WG<DH, BF>::template rs<1>(dv, pf[kc], make_smem_desc_sw128(udO + hq * 8192 + kc * 2048, 16384, 1024), 1u);
#pragma unroll
      for (int kc = 0; kc < 4; ++kc)
        WG<DH, BF>::template rs<1>(dk, df[kc], make_smem_desc_sw128(uQ + hq * 8192 + kc * 2048, 16384, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int e = 0; e < DH / 2; ++e) {
        reg_fence(dv[e]);
        reg_fence(dk[e]);
      }
#pragma unroll
      for (int kc = 0; kc < 4; ++kc)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          reg_fence(pf[kc][q]);
          reg_fence(df[kc][q]);
        }
      __syncthreads();  // both warpgroups' dS^T rows are in smem
      if (DH == 128 || wg == 0) {
        const int c0 = DH == 128 ? wg * 64 : 0;  // dh columns of dQ this warpgroup computes
        float dq[32];
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < 8; ++kc)  // contraction over the 128 keys
          WG<64, BF>::template ss<1, 1>(dq, make_smem_desc_sw128(udS + kc * 2048, 8192, 1024),
                                        make_smem_desc_sw128(uK + (c0 / 64) * 16384 + kc * 2048, 16384, 1024), kc > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int e = 0; e < 32; ++e) reg_fence(dq[e]);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int qi = i * 128 + hq * 64 + fr + 8 * r;
          if (qi < L) {
            const size_t base = ((size_t)b * L + qi) * ld3 + h * DH + c0 + fc;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              const float x0 = dq[4 * c + 2 * r], x1 = dq[4 * c + 2 * r + 1];
              if (a.dqkv16 != nullptr) {  // single key tile: final values, straight to the 16-bit GEMM operand
                *reinterpret_cast<uint32_t*>(a.dqkv16 + base + 8 * c) = cvt16x2(x0, x1, a.fmt_grad);
              } else if (a.dq_atomic) {
                atomicAdd(a.dqkv32 + base + 8 * c, x0);
                atomicAdd(a.dqkv32 + base + 8 * c + 1, x1);
              } else {
                *reinterpret_cast<float2*>(a.dqkv32 + base + 8 * c) = make_float2(x0, x1);
              }
            }
          }
        }
      }
      __syncthreads();  // dS^T buffer free for the next half
    }
  }
  // dK, dV of this key tile (rows = keys)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int kv = j * 128 + wg * 64 + fr + 8 * r;
    if (kv < L) {
      const size_t row = ((size_t)b * L + kv) * ld3 + h * DH + fc;
#pragma unroll
      for (int c = 0; c < DH / 8; ++c) {
        const float k0 = dk[4 * c + 2 * r], k1 = dk[4 * c + 2 * r + 1];
        const float v0 = dv[4 * c + 2 * r], v1 = dv[4 * c + 2 * r + 1];
        if (a.dqkv16 != nullptr) {
          *reinterpret_cast<uint32_t*>(a.dqkv16 + row + a.d + 8 * c) = cvt16x2(k0, k1, a.fmt_grad);
          *reinterpret_cast<uint32_t*>(a.dqkv16 + row + 2 * a.d + 8 * c) = cvt16x2(v0, v1, a.fmt_grad);
        } else {
          *reinterpret_cast<float2*>(a.dqkv32 + row + a.d + 8 * c) = make_float2(k0, k1);
          *reinterpret_cast<float2*>(a.dqkv32 + row + 2 * a.d + 8 * c) = make_float2(v0, v1);
        }
      }
    }
  }
}

template <int DH, int BF, int DROP>
static int launch_bwd_tc(const AttnBwdArgs& a, cudaStream_t stream) {
  using Cfg = AttnBwdCfg<DH>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attention_bwd_wgmma_kernel<DH, BF, DROP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(attention_bwd): %s", cudaGetErrorString(e));
      return (int)e;
    }
    attr_set = true;
  }
  dim3 grid((a.L + 127) / 128, a.H, a.B);
  launch_k(attention_bwd_wgmma_kernel<DH, BF, DROP>, dim3(grid), dim3(256), Cfg::kSmemBytes, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("attention_bwd launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

template <int DH, int BF>
static int launch_bwd_tc_drop(const AttnBwdArgs& a, cudaStream_t stream, int* kernel_used) {
  if (kernel_used) *kernel_used = (DH == 128 ? 4 : 0) + 2 * BF + (a.drop.on ? 1 : 0);
  return a.drop.on ? launch_bwd_tc<DH, BF, 1>(a, stream) : launch_bwd_tc<DH, BF, 0>(a, stream);
}

int launch_attention_bwd(const AttnBwdArgs& a, cudaStream_t stream, int* kernel_used) {
  if (kernel_used) *kernel_used = -1;
  if (a.fmt_act != a.fmt_grad) {
    set_error("launch_attention_bwd: activations and gradients must share one 16-bit format (got %d and %d)", a.fmt_act, a.fmt_grad);
    return (int)cudaErrorInvalidValue;
  }
  const bool bf = a.fmt_act != 0;
  if (a.dh == 128) return bf ? launch_bwd_tc_drop<128, 1>(a, stream, kernel_used) : launch_bwd_tc_drop<128, 0>(a, stream, kernel_used);
  if (a.dh == 64) return bf ? launch_bwd_tc_drop<64, 1>(a, stream, kernel_used) : launch_bwd_tc_drop<64, 0>(a, stream, kernel_used);
  set_error("launch_attention_bwd: tensor-core path needs dh in {64,128}, got %d", a.dh);
  return (int)cudaErrorInvalidValue;
}

}  // namespace uv
