// Multi-head attention core of the encoder layer (torch MHA semantics, SURVEY.md §A.3;
// call site model/transformer_encoder_droppath.py:118):
//     S = (Q K^T) / sqrt(dh) + key-padding(-inf);  P = softmax_j(S);  O = P V
// Q, K, V are the three d-wide column blocks of one [B*L, 3d] 16-bit matrix written by the in-projection GEMM.
// Flash-style: S and P never touch HBM.  wgmma path (dh in {64,128}):
//   CTA = one (batch, head, 128-query tile), two warpgroups of 64 query rows each; loop over 128-key tiles (K / V double-buffered
//   through TMA) with online softmax:
//     S  = Q K^T : wgmma m64n128, A = Q and B = K from 128B-swizzled K-major smem tiles, fp32 accumulators in registers
//     P  = exp2(scaled S - running max), converted in registers to 16-bit wgmma A fragments (the m64n128 accumulator layout
//          is the A-fragment layout of the next product, so P never leaves the registers)
//     O  = alpha O + P V : wgmma m64 x dh, A = P (registers), B = V (MN-major smem tile, dh contiguous)
// A SIMT kernel covers other head sizes (e.g. dh = 32 of the d=256 demo config).
#include <math.h>

#include "kernels.h"
#include "ptx.cuh"
#include "rowops.h"
#include "wgmma.cuh"

namespace uv {

// SPLIT (fp16x3): Q, K and V tiles are held as hi and lo planes.  For DH = 128 two K / V stages of both planes (256 KB) do not
// fit next to Q, so the split DH = 128 kernel single-buffers K / V (the next tile's load waits until the current one is done).
template <int DH, bool SPLIT = false>
struct AttnCfg {
  static constexpr int kPlanes = SPLIT ? 2 : 1;
  static constexpr int kStages = (SPLIT && DH == 128) ? 1 : 2;
  static constexpr int kQPlane = 128 * DH * 2;            // DH/64 boxes of [128 rows x 64]
  static constexpr int kQBytes = kPlanes * kQPlane;
  static constexpr int kKVBytes = 128 * DH * 2;           // one plane of one K or V tile, same boxes
  static constexpr int kSmemBytes = 1024 + kQBytes + 2 * kStages * kPlanes * kKVBytes + 2 * 128 * 4 + 64;
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// DROP = 1: attention dropout.  The multipliers of the tile are generated while the S product runs (one Philox call per 8
// elements) and kept as keep-bits; P o M is what feeds P V, while the row sum, the running max and lse stay un-dropped.
// CAUSAL = 1: query row i sees keys j <= i only (the additive triu(-inf) mask of CLIP's text transformer).  Key tiles that lie
// wholly above the diagonal are not loaded, and masked scores enter the softmax as -inf, so they contribute exactly 0.
template <int DH, int BF, int DROP, int CAUSAL>
__device__ __forceinline__ void attention_tile(const AttnArgs& a) {
  using Cfg = AttnCfg<DH>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::kQBytes;          // [2] K tiles
  uint8_t* sV = sK + 2 * Cfg::kKVBytes;     // [2] V tiles
  float* s_bias = reinterpret_cast<float*>(sV + 2 * Cfg::kKVBytes);  // [2][128] 0 or -inf per key of the tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_bias + 2 * 128);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;  // [2]

  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;               // query rows [64 wg, 64 wg + 64) of the tile
  const int tid = threadIdx.x & 127;
  const int fr = 16 * (tid >> 5) + (lane >> 2);  // accumulator rows fr, fr + 8; columns 8 i + fc, + 1
  const int fc = 2 * (lane & 3);
  const int q0 = blockIdx.x * 128;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int L = a.L;
  const int num_kv = CAUSAL ? min((L + 127) / 128, q0 / 128 + 1) : (L + 127) / 128;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&a.tm_qkv);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // barriers are set up; from here on the kernel reads what the previous kernels wrote
  const DropSpec drop = drop_resolve(a.drop);  // (the seed is read after the PDL wait: a preceding kernel may write it)

  auto load_kv = [&](int j) {
    const int s = j & 1;
    mbar_arrive_expect_tx(&kv_full[s], 2 * Cfg::kKVBytes);
#pragma unroll
    for (int kb = 0; kb < DH / 64; ++kb) {
      tma_load_2d(sK + s * Cfg::kKVBytes + kb * 16384, &a.tm_qkv, &kv_full[s], a.d + h * DH + kb * 64, b * L + j * 128);
      tma_load_2d(sV + s * Cfg::kKVBytes + kb * 16384, &a.tm_qkv, &kv_full[s], 2 * a.d + h * DH + kb * 64, b * L + j * 128);
    }
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(q_full, Cfg::kQBytes);
#pragma unroll
    for (int kb = 0; kb < DH / 64; ++kb) tma_load_2d(sQ + kb * 16384, &a.tm_qkv, q_full, h * DH + kb * 64, b * L + q0);
    load_kv(0);
  }

  const float kLog2e = 1.4426950408889634f * a.scale;  // scores are scaled by 1/sqrt(dh) inside the exponent
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // l_run: this thread's columns only (quad-summed at the end)
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;

  for (int j = 0; j < num_kv; ++j) {
    const int s = j & 1;
    __syncthreads();  // every wgmma of tile j-1 has retired: its K / V buffers and bias row may be overwritten
    if (threadIdx.x == 0 && j + 1 < num_kv) load_kv(j + 1);
    if (threadIdx.x < 128) {
      const int key = j * 128 + threadIdx.x;
      s_bias[s * 128 + threadIdx.x] = (key < L && a.key_mask[(size_t)b * L + key] != 0.f) ? 0.f : -INFINITY;
    }
    __syncthreads();
    if (j == 0) mbar_wait(q_full, 0);
    mbar_wait(&kv_full[s], (j >> 1) & 1);
    const uint32_t kbase = smem_u32(sK + s * Cfg::kKVBytes), vbase = smem_u32(sV + s * Cfg::kKVBytes);

    float sacc[64];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < DH / 16; ++ks) {
      const uint32_t off = (ks / 4) * 16384 + (ks % 4) * 32;
      WG<128, BF>::template ss<0, 0>(sacc, make_smem_desc_sw128(smem_u32(sQ) + wg * 8192 + off, 16, 1024),
                                     make_smem_desc_sw128(kbase + off, 16, 1024), ks > 0 ? 1u : 0u);
    }
    wgmma_commit();
    // keep-bits of this thread's 64 probabilities of the tile: fragment (kc, q), element e -> bit 8 (kc & 3) + 2 q + e of
    // mb[kc >> 2].  Query rows fr / fr + 8 and keys 16 kc + fc + {0, 1, 8, 9} are exactly one attn_drop_block call.
    uint32_t mb[2] = {0u, 0u};
    if constexpr (DROP != 0) {
      const unsigned int bh = (unsigned int)(b * a.H + h), i0 = (unsigned int)(q0 + wg * 64 + fr);
#pragma unroll
      for (int kc = 0; kc < 8; ++kc) {
        const uint4 rr = attn_drop_block(drop, bh, i0, (unsigned int)(j * 128 + 16 * kc + fc));
        const uint32_t w[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t wq = w[2 * (q & 1) + (q >> 1)];  // row bit 3 = q & 1, key bit 3 = q >> 1
          mb[kc >> 2] |= ((wq & 0xffffu) >= drop.thresh ? 1u : 0u) << (8 * (kc & 3) + 2 * q);
          mb[kc >> 2] |= ((wq >> 16) >= drop.thresh ? 1u : 0u) << (8 * (kc & 3) + 2 * q + 1);
        }
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 64; ++i) reg_fence(sacc[i]);

    // online softmax over this tile's 128 keys (log2 units)
    const float* bias = s_bias + s * 128;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float x = sacc[4 * i + e] * kLog2e + bias[8 * i + fc + (e & 1)];
        if constexpr (CAUSAL != 0) {
          if (j * 128 + 8 * i + fc + (e & 1) > q0 + wg * 64 + fr + 8 * (e >> 1)) x = -INFINITY;
        }
        sacc[4 * i + e] = x;
        mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m_new = fmaxf(m_run[r], quad_max(mx[r]));
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[r] = exp2f(m_run[r] - m_use[r]);  // m_run = -inf -> 0
      m_run[r] = m_new;
    }
    float psum[2] = {0.f, 0.f};
    uint32_t pf[8][4];  // P as wgmma A fragments: k-chunk kc = keys [16 kc, 16 kc + 16)
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = q & 1;  // fragment register q: row fr (+8 for odd q), keys 16 kc + 8 (q >> 1) + fc, + 1
        const float p0 = exp2f(sacc[8 * kc + 2 * q] - m_use[r]);
        const float p1 = exp2f(sacc[8 * kc + 2 * q + 1] - m_use[r]);
        psum[r] += p0 + p1;
        if constexpr (DROP != 0) {
          const uint32_t bits = mb[kc >> 2] >> (8 * (kc & 3) + 2 * q);
          pf[kc][q] = cvt16x2((bits & 1u) ? p0 * drop.scale : 0.f, (bits & 2u) ? p1 * drop.scale : 0.f, BF);
        } else {
          pf[kc][q] = cvt16x2(p0, p1, BF);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + psum[r];
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
      o[4 * i] *= alpha[0];
      o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1];
      o[4 * i + 3] *= alpha[1];
    }
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 8; ++kc)  // V tile: 64-wide dh blocks of [128 kv rows x 128 B]; 16 kv rows = two 1024 B swizzle atoms
      WG<DH, BF>::template rs<1>(o, pf[kc], make_smem_desc_sw128(vbase + kc * 2048, 16384, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) reg_fence(o[i]);
#pragma unroll
    for (int kc = 0; kc < 8; ++kc)
#pragma unroll
      for (int q = 0; q < 4; ++q) reg_fence(pf[kc][q]);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = q0 + wg * 64 + fr + 8 * r;
    const float l = quad_sum(l_run[r]);
    if (qi < L) {
      const float inv = 1.f / l;
      uint16_t* dst = a.out + ((size_t)b * L + qi) * a.d + h * DH + fc;
#pragma unroll
      for (int i = 0; i < DH / 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + 8 * i) = cvt16x2(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv, BF);
      if (a.lse && (lane & 3) == 0) a.lse[((size_t)b * a.H + h) * L + qi] = m_run[r] * 0.6931471805599453f + logf(l);
    }
  }
}

template <int DH, int BF, int DROP>
__global__ void __launch_bounds__(256, 1) attention_wgmma_kernel(const __grid_constant__ AttnArgs a) {
  attention_tile<DH, BF, DROP, 0>(a);
}

// dh = 64 with the causal mask (inference, no dropout): CLIP's text transformer.
template <int BF>
__global__ void __launch_bounds__(256, 1) attention_wgmma_causal_kernel(const __grid_constant__ AttnArgs a) {
  attention_tile<64, BF, 0, 1>(a);
}

// fp16x3 attention (inference, no dropout).  tm_qkv is a plane pair; S takes Q_hi K_hi + Q_lo K_hi + Q_hi K_lo, P is split in registers
// into hi and lo A fragments and O += P_hi V_hi + P_lo V_hi + P_hi V_lo.  The row sum, running max and lse stay fp32.
// A kernel of its own, so that the fp16 / bf16 kernels above are compiled exactly as before.
template <int DH>
__global__ void __launch_bounds__(256, 1) attention_wgmma_split_kernel(const __grid_constant__ AttnArgs a) {
  using Cfg = AttnCfg<DH, true>;
  constexpr int BF = 0, NP = Cfg::kPlanes, NS = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::kQBytes;          // [NS][NP] K tiles
  uint8_t* sV = sK + NS * NP * Cfg::kKVBytes;  // [NS][NP] V tiles
  float* s_bias = reinterpret_cast<float*>(sV + NS * NP * Cfg::kKVBytes);  // [2][128] 0 or -inf per key of the tile
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_bias + 2 * 128);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;  // [2]

  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;               // query rows [64 wg, 64 wg + 64) of the tile
  const int tid = threadIdx.x & 127;
  const int fr = 16 * (tid >> 5) + (lane >> 2);  // accumulator rows fr, fr + 8; columns 8 i + fc, + 1
  const int fc = 2 * (lane & 3);
  const int q0 = blockIdx.x * 128;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int L = a.L;
  const int num_kv = (L + 127) / 128;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&a.tm_qkv);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();  // barriers are set up; from here on the kernel reads what the previous kernels wrote

  auto load_kv = [&](int j) {
    const int s = NS == 2 ? (j & 1) : 0;
    mbar_arrive_expect_tx(&kv_full[s], 2 * NP * Cfg::kKVBytes);  // K and V, every plane
#pragma unroll
    for (int kb = 0; kb < DH / 64; ++kb) {
#pragma unroll
      for (int pl = 0; pl < NP; ++pl) {
        tma_load_3d(sK + (s * NP + pl) * Cfg::kKVBytes + kb * 16384, &a.tm_qkv, &kv_full[s], a.d + h * DH + kb * 64, b * L + j * 128, pl);
        tma_load_3d(sV + (s * NP + pl) * Cfg::kKVBytes + kb * 16384, &a.tm_qkv, &kv_full[s], 2 * a.d + h * DH + kb * 64, b * L + j * 128, pl);
      }
    }
  };
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(q_full, Cfg::kQBytes);
#pragma unroll
    for (int kb = 0; kb < DH / 64; ++kb)
#pragma unroll
      for (int pl = 0; pl < NP; ++pl) tma_load_3d(sQ + pl * Cfg::kQPlane + kb * 16384, &a.tm_qkv, q_full, h * DH + kb * 64, b * L + q0, pl);
    load_kv(0);
  }

  const float kLog2e = 1.4426950408889634f * a.scale;  // scores are scaled by 1/sqrt(dh) inside the exponent
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // l_run: this thread's columns only (quad-summed at the end)
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;

  for (int j = 0; j < num_kv; ++j) {
    const int s = j & 1;  // bias row; also the K / V stage unless NS == 1
    const int skv = NS == 2 ? s : 0;
    __syncthreads();  // every wgmma of tile j-1 has retired: its K / V buffers and bias row may be overwritten
    if (threadIdx.x == 0) {
      if constexpr (NS == 2) {
        if (j + 1 < num_kv) load_kv(j + 1);
      } else {
        if (j > 0) load_kv(j);  // single buffer: tile j replaces tile j - 1 now that it is done
      }
    }
    if (threadIdx.x < 128) {
      const int key = j * 128 + threadIdx.x;
      s_bias[s * 128 + threadIdx.x] = (key < L && a.key_mask[(size_t)b * L + key] != 0.f) ? 0.f : -INFINITY;
    }
    __syncthreads();
    if (j == 0) mbar_wait(q_full, 0);
    mbar_wait(&kv_full[skv], NS == 2 ? ((j >> 1) & 1) : (j & 1));
    const uint32_t kbase = smem_u32(sK + skv * NP * Cfg::kKVBytes), vbase = smem_u32(sV + skv * NP * Cfg::kKVBytes);

    float sacc[64];
    wgmma_fence();
#pragma unroll
    for (int pr = 0; pr < 3; ++pr) {  // (Q hi, K hi), (Q lo, K hi), (Q hi, K lo)
      const uint32_t qb = smem_u32(sQ) + (pr == 1 ? Cfg::kQPlane : 0), kb_ = kbase + (pr == 2 ? Cfg::kKVBytes : 0);
#pragma unroll
      for (int ks = 0; ks < DH / 16; ++ks) {
        const uint32_t off = (ks / 4) * 16384 + (ks % 4) * 32;
        WG<128, BF>::template ss<0, 0>(sacc, make_smem_desc_sw128(qb + wg * 8192 + off, 16, 1024),
                                       make_smem_desc_sw128(kb_ + off, 16, 1024), (pr > 0 || ks > 0) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 64; ++i) reg_fence(sacc[i]);

    // online softmax over this tile's 128 keys (log2 units)
    const float* bias = s_bias + s * 128;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float x = sacc[4 * i + e] * kLog2e + bias[8 * i + fc + (e & 1)];
        sacc[4 * i + e] = x;
        mx[e >> 1] = fmaxf(mx[e >> 1], x);
      }
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m_new = fmaxf(m_run[r], quad_max(mx[r]));
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[r] = exp2f(m_run[r] - m_use[r]);  // m_run = -inf -> 0
      m_run[r] = m_new;
    }
    float psum[2] = {0.f, 0.f};
    uint32_t pf[8][4], pfl[8][4];  // P = hi + lo as wgmma A fragments: k-chunk kc = keys [16 kc, 16 kc + 16)
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = q & 1;  // fragment register q: row fr (+8 for odd q), keys 16 kc + 8 (q >> 1) + fc, + 1
        const float p0 = exp2f(sacc[8 * kc + 2 * q] - m_use[r]);
        const float p1 = exp2f(sacc[8 * kc + 2 * q + 1] - m_use[r]);
        psum[r] += p0 + p1;
        pf[kc][q] = cvt16x2(p0, p1, BF);
        pfl[kc][q] = cvt16x2_lo(p0, p1);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + psum[r];
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
      o[4 * i] *= alpha[0];
      o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1];
      o[4 * i + 3] *= alpha[1];
    }
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {  // V tile: 64-wide dh blocks of [128 kv rows x 128 B]; 16 kv rows = two 1024 B swizzle atoms
      WG<DH, BF>::template rs<1>(o, pf[kc], make_smem_desc_sw128(vbase + kc * 2048, 16384, 1024), 1u);
      WG<DH, BF>::template rs<1>(o, pfl[kc], make_smem_desc_sw128(vbase + kc * 2048, 16384, 1024), 1u);
      WG<DH, BF>::template rs<1>(o, pf[kc], make_smem_desc_sw128(vbase + Cfg::kKVBytes + kc * 2048, 16384, 1024), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) reg_fence(o[i]);
#pragma unroll
    for (int kc = 0; kc < 8; ++kc)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        reg_fence(pf[kc][q]);
        reg_fence(pfl[kc][q]);
      }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = q0 + wg * 64 + fr + 8 * r;
    const float l = quad_sum(l_run[r]);
    if (qi < L) {
      const float inv = 1.f / l;
      uint16_t* dst = a.out + ((size_t)b * L + qi) * a.d + h * DH + fc;
#pragma unroll
      for (int i = 0; i < DH / 8; ++i) {
        *reinterpret_cast<uint32_t*>(dst + 8 * i) = cvt16x2(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv, BF);
        *reinterpret_cast<uint32_t*>(dst + a.lo_out + 8 * i) = cvt16x2_lo(o[4 * i + 2 * r] * inv, o[4 * i + 2 * r + 1] * inv);
      }
      if (a.lse && (lane & 3) == 0) a.lse[((size_t)b * a.H + h) * L + qi] = m_run[r] * 0.6931471805599453f + logf(l);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// SIMT attention for head sizes the tensor-core kernel does not tile (dh not in {64,128}).
// One warp per (b, h, query row); scores staged in shared memory.
// ------------------------------------------------------------------------------------------------
struct AttnSimtArgs {
  const uint16_t* qkv;  // [B*L, 3d]
  const float* key_mask;
  uint16_t* out;
  float* lse;
  float scale;
  int B, L, H, dh, d, fmt;
  DropSpec drop;
  long long lo_qkv, lo_out;  // SPLIT: elements from qkv / out to their lo planes
};

// DROP = 1: attention dropout, one Philox call per element (attn_drop_mul1); p o m is rounded to 16 bit where p is otherwise.
// SPLIT: fp16x3 - Q, K and V are read as hi + lo in fp32, p is rounded to hi + lo as the split tensor-core path rounds it, and
// the output is written as a hi / lo pair.
template <int DROP, bool SPLIT = false>
__global__ void __launch_bounds__(128) attention_simt_kernel(const AttnSimtArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  extern __shared__ float s_sc[];  // [4 warps][L]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * 4 + warp;
  if (gw >= a.B * a.H * a.L) return;
  const int i = gw % a.L;
  const int h = (gw / a.L) % a.H;
  const int b = gw / (a.L * a.H);
  float* sc = s_sc + warp * a.L;
  const size_t ld = (size_t)3 * a.d;
  const uint16_t* qrow = a.qkv + ((size_t)b * a.L + i) * ld + h * a.dh;
  float mx = -INFINITY;
  for (int j = lane; j < a.L; j += 32) {
    float s = -INFINITY;
    if (a.key_mask[(size_t)b * a.L + j] != 0.f) {
      const uint16_t* krow = a.qkv + ((size_t)b * a.L + j) * ld + a.d + h * a.dh;
      s = 0.f;
      if constexpr (SPLIT) {
        for (int c = 0; c < a.dh; ++c) s += ld16x3(qrow[c], qrow[a.lo_qkv + c]) * ld16x3(krow[c], krow[a.lo_qkv + c]);
      } else {
        for (int c = 0; c < a.dh; ++c) s += ld16(qrow[c], a.fmt) * ld16(krow[c], a.fmt);
      }
      s *= a.scale;
    }
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  const float m_use = (mx == -INFINITY) ? 0.f : mx;
  float sum = 0.f;
  for (int j = lane; j < a.L; j += 32) {
    const float p = expf(sc[j] - m_use);
    sum += p;
    float pm = p;
    if constexpr (DROP != 0) pm = p * attn_drop_mul1(drop, (unsigned int)(b * a.H + h), (unsigned int)i, (unsigned int)j);
    if constexpr (SPLIT) sc[j] = ld16x3(cvt16(pm, 0), cvt16_lo(pm));
    else sc[j] = ld16(cvt16(pm, a.fmt), a.fmt);  // same operand rounding as the tensor-core path
  }
  sum = warp_sum(sum);
  __syncwarp();
  for (int c = lane; c < a.dh; c += 32) {
    const uint16_t* vcol = a.qkv + (size_t)b * a.L * ld + 2 * a.d + h * a.dh + c;
    float o = 0.f;
    if constexpr (SPLIT) {
      for (int j = 0; j < a.L; ++j) o += sc[j] * ld16x3(vcol[(size_t)j * ld], vcol[a.lo_qkv + (size_t)j * ld]);
      a.out[a.lo_out + ((size_t)b * a.L + i) * a.d + h * a.dh + c] = cvt16_lo(o / sum);
    } else {
      for (int j = 0; j < a.L; ++j) o += sc[j] * ld16(vcol[(size_t)j * ld], a.fmt);
    }
    a.out[((size_t)b * a.L + i) * a.d + h * a.dh + c] = cvt16(o / sum, a.fmt);
  }
  if (lane == 0 && a.lse) a.lse[((size_t)b * a.H + h) * a.L + i] = mx + logf(sum);
}

template <int DH, int BF, int DROP>
static int launch_tc(const AttnArgs& a, cudaStream_t stream) {
  using Cfg = AttnCfg<DH>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e =
        cudaFuncSetAttribute(attention_wgmma_kernel<DH, BF, DROP>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(attention): %s", cudaGetErrorString(e));
      return (int)e;
    }
    attr_set = true;
  }
  dim3 grid((a.L + 127) / 128, a.H, a.B);
  launch_k(attention_wgmma_kernel<DH, BF, DROP>, dim3(grid), dim3(256), Cfg::kSmemBytes, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("attention launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

template <int BF>
static int launch_tc_causal(const AttnArgs& a, cudaStream_t stream) {
  using Cfg = AttnCfg<64>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attention_wgmma_causal_kernel<BF>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(attention, causal): %s", cudaGetErrorString(e));
      return (int)e;
    }
    attr_set = true;
  }
  dim3 grid((a.L + 127) / 128, a.H, a.B);
  launch_k(attention_wgmma_causal_kernel<BF>, dim3(grid), dim3(256), Cfg::kSmemBytes, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("attention launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

template <int DH>
static int launch_tc_split(const AttnArgs& a, cudaStream_t stream) {
  using Cfg = AttnCfg<DH, true>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attention_wgmma_split_kernel<DH>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(attention, fp16x3): %s", cudaGetErrorString(e));
      return (int)e;
    }
    attr_set = true;
  }
  dim3 grid((a.L + 127) / 128, a.H, a.B);
  launch_k(attention_wgmma_split_kernel<DH>, dim3(grid), dim3(256), Cfg::kSmemBytes, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("attention launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

template <int DH, int BF>
static int launch_tc_drop(const AttnArgs& a, cudaStream_t stream) {
  return a.drop.on ? launch_tc<DH, BF, 1>(a, stream) : launch_tc<DH, BF, 0>(a, stream);
}

int launch_attention_simt(const AttnArgs& a, const uint16_t* qkv, cudaStream_t stream, int* kernel_used) {
  AttnSimtArgs s{qkv, a.key_mask, a.out, a.lse, a.scale, a.B, a.L, a.H, a.dh, a.d, a.fmt, a.drop, a.lo_qkv, a.lo_out};
  const int warps = a.B * a.H * a.L;
  const size_t smem = (size_t)4 * a.L * sizeof(float);
  if (a.split && (a.fmt != 0 || a.drop.on)) {
    set_error("attention_simt: fp16x3 needs fmt 0 and no dropout");
    return (int)cudaErrorInvalidValue;
  }
  auto kern = a.split ? attention_simt_kernel<0, true> : a.drop.on ? attention_simt_kernel<1> : attention_simt_kernel<0>;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("attention_simt smem %zu: %s", smem, cudaGetErrorString(e));
      return (int)e;
    }
  }
  launch_k(kern, dim3((warps + 3) / 4), dim3(128), smem, stream, s);
  if (kernel_used) *kernel_used = a.split ? ATT_SIMT_SPLIT : a.drop.on ? ATT_SIMT_DROP : ATT_SIMT;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("attention_simt launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

int launch_attention(const AttnArgs& a, cudaStream_t stream, int* kernel_used) {
  if (a.causal) {
    if (a.dh != 64 || a.split || a.drop.on) {
      set_error("launch_attention: the causal mask needs dh = 64, fp16 or bf16 operands and no dropout");
      return (int)cudaErrorInvalidValue;
    }
    if (kernel_used) *kernel_used = ATT_CAUSAL + (a.fmt ? 1 : 0);
    return a.fmt ? launch_tc_causal<1>(a, stream) : launch_tc_causal<0>(a, stream);
  }
  if (a.split) {
    if (a.fmt != 0 || a.drop.on) {
      set_error("launch_attention: fp16x3 needs fmt 0 and no dropout");
      return (int)cudaErrorInvalidValue;
    }
    if (kernel_used) *kernel_used = a.dh == 128 ? ATT_SPLIT128 : ATT_SPLIT64;
    if (a.dh == 128) return launch_tc_split<128>(a, stream);
    if (a.dh == 64) return launch_tc_split<64>(a, stream);
  }
  if (kernel_used) *kernel_used = ATT_TC + (a.dh == 128 ? 4 : 0) + (a.fmt ? 2 : 0) + (a.drop.on ? 1 : 0);
  if (a.dh == 128) return a.fmt ? launch_tc_drop<128, 1>(a, stream) : launch_tc_drop<128, 0>(a, stream);
  if (a.dh == 64) return a.fmt ? launch_tc_drop<64, 1>(a, stream) : launch_tc_drop<64, 0>(a, stream);
  if (kernel_used) *kernel_used = -1;
  set_error("launch_attention: tensor-core path needs dh in {64,128}, got %d", a.dh);
  return (int)cudaErrorInvalidValue;
}

// The attention-dropout multipliers of `spec` as dense [B, H, L, L] (parity tests; the kernels above never store them).
__global__ void __launch_bounds__(256) attention_dropout_mask_kernel(const DropSpec spec_in, int L, size_t n, float* __restrict__ out) {
  pdl_prologue();
  const DropSpec spec = drop_resolve(spec_in);
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
    const unsigned int j = (unsigned int)(idx % L), i = (unsigned int)((idx / L) % L), bh = (unsigned int)(idx / ((size_t)L * L));
    out[idx] = attn_drop_mul1(spec, bh, i, j);
  }
}

int launch_attention_dropout_mask(const DropSpec& spec, int B, int H, int L, float* out, cudaStream_t stream) {
  const size_t n = (size_t)B * H * L * L;
  const unsigned int blocks = (unsigned int)((n + 255) / 256 < 65536 ? (n + 255) / 256 : 65536);
  launch_k(attention_dropout_mask_kernel, dim3(blocks), dim3(256), 0, stream, spec, L, n, out);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("attention_dropout_mask launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

}  // namespace uv
