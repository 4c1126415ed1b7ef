// Persistent, warp-specialised wgmma GEMM for sm_90a with a fused, run-time configured epilogue.
//
//   C[M,N] = epilogue( sum_k A[m,k] * B[n,k] ),  A/B 16-bit (fp16 or bf16, both operands in one format), fp32 accumulation.
//
// This one kernel serves every dense contraction of the UniVTG hot path (SURVEY.md §2.2 rows K1-K3, K5, K7,
// K9-K11 and their backward passes): input projectors (model/univtg.py:399-406), the three attention
// in-projections + out-projection (torch MHA called at model/transformer_encoder_droppath.py:118), the FFN
// (:122) and the k=3 Conv1d heads (model/univtg.py:378-382) expressed as three row-shifted K segments.
//
// Roles (384 threads = 3 warpgroups, 1 CTA / SM, persistent over a static, longest-first deal of 128 x BN tiles):
//   warpgroup 2 (one elected lane of warp 8): TMA producer (cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier
//                    expect_tx); it gives most of its registers to the consumers (setmaxnreg)
//   warpgroups 0, 1: consumers.  Each issues wgmma m64 x BN x k16 for its 64 rows of the tile (accumulators in registers),
//                    then runs the epilogue of those rows: the accumulators go through shared memory 32 columns at a time so
//                    that a thread owns 16 consecutive columns of one row (whole 32 B sectors, 128-bit global accesses).
// CL = 2 (clusters of two CTAs, K-major B only): the pair computes two vertically adjacent 128-row tiles of the same BN
// columns; each CTA loads half of the B tile and multicasts it to both, so every B byte crosses L2 once per pair.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "kernels.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace uv {

// The tile width BN is a launch argument, checked by launch_gemm_group: a multiple of 16 in [32, 256]; a multiple of 32 for 2-CTA
// clusters, which need a K-major B; a multiple of 64 when B is MN-major (CL = 1 only).  The host picks it per launch so that the
// tile count fills the SMs with as little wave quantisation as possible; the consumers dispatch on it once (consumer_tiles<BN>),
// and only the widths above are compiled.
// Operand ring: kRingBytes of shared memory cut into as many stages as the tile width allows (a stage = the 16 KB A tile + BN x
// 128 B of B), at most kMaxStages.
template <int CL>
struct GemmCfg {
  static constexpr int kMaxStages = 8;
  static constexpr int kABytes = GEMM_BM * 128;                 // 128 rows x 64 x 2 B
  static constexpr int kRingBytes = 4 * (kABytes + 256 * 128);  // 192 KB
  static constexpr int kEpiStride = 36;                         // floats per staged accumulator row (32 columns + 4 pad)
  static constexpr int kEpiFloats = 2 * 64 * kEpiStride;        // one 64 x 32 staging tile per consumer warpgroup
  static constexpr int kSmemBytes = 1024 /*align slack*/ + kRingBytes + kEpiFloats * 4 + 256;
  __host__ __device__ static constexpr int stage_bytes(int bn) { return kABytes + bn * 128; }  // multiple of 1024 (bn % 16 == 0)
  __host__ __device__ static constexpr int num_stages(int bn) {
    return kRingBytes / stage_bytes(bn) < kMaxStages ? kRingBytes / stage_bytes(bn) : kMaxStages;
  }
};

constexpr int kGemmThreads = 384;  // two consumer warpgroups + the producer warpgroup

struct TileInfo {
  int p, m_blk, n_blk, kb0, kb1, split;
};

// `t` is a unit index of the deal (gemm_deal_unit, kernels.h): problems in order (launch_gemm_group put them in deal order),
// then tile order inside the problem.  CL = 1: a unit is one tile.  CL = 2: a unit is a 256-row PAIR tile made of two vertically adjacent 128-row tiles
// (m_blk = 2*pair + rank, same n_blk).  The odd tail tile of a problem is a phantom whose rows are all out of range.
template <int CL, bool SPLIT>
__host__ __device__ __forceinline__ bool decode_tile(const GemmGroup& g, int bn, int t, int rank, TileInfo& ti) {
  for (int p = 0; p < g.num; ++p) {
    const GemmProblem& pr = g.p[p];
    const int tm_real = (pr.M + GEMM_BM - 1) / GEMM_BM;
    const int tm = (tm_real + CL - 1) / CL;
    const int tn = (pr.N + bn - 1) / bn;
    const int cnt = tm * tn * pr.ksplit;
    if (t < cnt) {
      ti.p = p;
      ti.n_blk = t % tn;
      const int rest = t / tn;
      ti.m_blk = (rest % tm) * CL + rank;
      ti.split = rest / tm;
      const int total_kb = pr.taps * pr.kblk_per_tap * (SPLIT ? 3 : 1);
      const int per = gemm_unit_kblocks(pr, SPLIT);
      ti.kb0 = ti.split * per;
      ti.kb1 = total_kb < ti.kb0 + per ? total_kb : ti.kb0 + per;
      return true;
    }
    t -= cnt;
  }
  return false;
}

__device__ __forceinline__ void stamp(unsigned long long* dbg, int slot) {
  if (dbg != nullptr) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    dbg[(size_t)blockIdx.x * 8 + slot] = t;
  }
}

// ---- mainloop: one 64-wide k-block of the warpgroup's 64 x N tile ----
// N is cut into wgmma widths 256 / 128 / 64 / 32 / 16 (largest first); slice [OFF, OFF + W) accumulates into acc[OFF/2 ...],
// which keeps the register layout of one m64nN accumulator.
template <int N, int OFF, int BF, int TA, int TB>
__device__ __forceinline__ void mma_cols(float* acc, uint64_t da, uint64_t db, uint32_t scale_d) {
  constexpr int W = N >= 256 ? 256 : N >= 128 ? 128 : N >= 64 ? 64 : N >= 32 ? 32 : 16;
  WG<W, BF>::template ss<TA, TB>(acc + OFF / 2, da, db, scale_d);
  if constexpr (N > W) {
    // next slice of B: K-major rows are 128 B apart; MN-major 64-wide blocks 8 KB apart (W is then a multiple of 64)
    constexpr uint32_t adv = TB ? (W / 64) * 8192 / 16 : W * 128 / 16;
    mma_cols<N - W, OFF + W, BF, TA, TB>(acc, da, db + adv, scale_d);
  }
}

// The consumer's view of the operand ring: where the stages are and which stage / phase it waits on next.
struct Ring {
  uint8_t* base;
  uint64_t* full;
  uint64_t* empty;
  int stage_bytes, stages;
  int stage;
  uint32_t phase;
};

template <int CL>
__device__ __forceinline__ void release_stage(const Ring& ring, int s, int tid, int crank) {
  // this warpgroup is done with stage s (in every CTA the stage was multicast from)
  if (tid == 0) {
    mbar_arrive(&ring.empty[s]);
    if (CL > 1) mbar_arrive_cluster(mapa_shared(smem_u32(&ring.empty[s]), (uint32_t)(crank ^ 1)));
  }
}

// k-blocks [kb0, kb1) of one tile into acc (BN / 2 floats: one m64nBN accumulator).  Width, operand format and both layouts are
// template parameters, so each combination gets a k-loop of its own; with a run-time choice inside the k-loop ptxas cannot keep
// more than one wgmma in flight.
template <int CL, int BN, int BF, int TA, int TB>
__device__ __forceinline__ void tile_mainloop(float* acc, Ring& ring, int kb0, int kb1, int cw, int tid, int crank) {
  // descriptor = constant high part (layout, LBO/SBO) + start address; one k-step of 16 elements advances the address by 32 B
  // inside the 128 B swizzle span (K-major) or by two 1024 B swizzle atoms (MN-major), in 16-byte units
  const uint64_t da_hi = TA ? make_smem_desc_sw128(0, 8192, 1024) : make_smem_desc_sw128(0, 16, 1024);
  const uint64_t db_hi = TB ? make_smem_desc_sw128(0, 8192, 1024) : make_smem_desc_sw128(0, 16, 1024);
  constexpr uint32_t a_step = TA ? 128u : 2u, b_step = TB ? 128u : 2u;
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&ring.full[ring.stage], ring.phase);
    const uint32_t sa = smem_u32(ring.base + ring.stage * ring.stage_bytes);
    // this warpgroup's 64 rows of A: K-major rows 64 cw.. (64 x 128 B); MN-major the cw-th 64-wide M block (8 KB each)
    const uint64_t da = da_hi + (uint64_t)((sa + cw * 8192) >> 4);
    const uint64_t db = db_hi + (uint64_t)((sa + GemmCfg<CL>::kABytes) >> 4);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GEMM_BK / 16; ++k)
      mma_cols<BN, 0, BF, TA, TB>(acc, da + k * a_step, db + k * b_step, (kb > kb0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
    if (prev >= 0) release_stage<CL>(ring, prev, tid, crank);
    prev = ring.stage;
    if (++ring.stage == ring.stages) {
      ring.stage = 0;
      ring.phase ^= 1;
    }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
  if (prev >= 0) release_stage<CL>(ring, prev, tid, crank);
}

// Operand format and layouts are per problem: pick the k-loop once per tile.  fp16x3 groups are K-major fp16 only, clusters
// need a K-major B and MN-major B needs BN % 64 == 0 (all checked on the host), so only those k-loops are compiled.
template <int CL, bool SPLIT, int BN>
__device__ __forceinline__ void tile_mainloop_any(float* acc, Ring& ring, int bf, int a_mn, int b_mn, int kb0, int kb1, int cw, int tid,
                                                  int crank) {
  if constexpr (SPLIT) {
    tile_mainloop<CL, BN, 0, 0, 0>(acc, ring, kb0, kb1, cw, tid, crank);
  } else {
    if constexpr (CL == 1 && BN % 64 == 0) {
      if (b_mn) {
        if (bf) {
          if (a_mn) tile_mainloop<CL, BN, 1, 1, 1>(acc, ring, kb0, kb1, cw, tid, crank);
          else tile_mainloop<CL, BN, 1, 0, 1>(acc, ring, kb0, kb1, cw, tid, crank);
        } else {
          if (a_mn) tile_mainloop<CL, BN, 0, 1, 1>(acc, ring, kb0, kb1, cw, tid, crank);
          else tile_mainloop<CL, BN, 0, 0, 1>(acc, ring, kb0, kb1, cw, tid, crank);
        }
        return;
      }
    }
    if (bf) {
      if (a_mn) tile_mainloop<CL, BN, 1, 1, 0>(acc, ring, kb0, kb1, cw, tid, crank);
      else tile_mainloop<CL, BN, 1, 0, 0>(acc, ring, kb0, kb1, cw, tid, crank);
    } else {
      if (a_mn) tile_mainloop<CL, BN, 0, 1, 0>(acc, ring, kb0, kb1, cw, tid, crank);
      else tile_mainloop<CL, BN, 0, 0, 0>(acc, ring, kb0, kb1, cw, tid, crank);
    }
  }
}

// ---- epilogue of one 16-column step of one row ----
struct EpiRow {
  bool valid;
  float rsc;
  const float* resid_row;
  const float* aux_row;
  const uint16_t* mask_row;
  const float* add_row;
  float* o32_row;
  float* o32i_row;
  uint16_t* o16_row;
  uint16_t* o16p_row;
  float* pre_row;
  uint16_t* dact_row;
};

__device__ __forceinline__ void ld16f(const float* p, float (&v)[16]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 t4 = reinterpret_cast<const float4*>(p)[q];
    v[4 * q] = t4.x; v[4 * q + 1] = t4.y; v[4 * q + 2] = t4.z; v[4 * q + 3] = t4.w;
  }
}

// FULL = false drops the training-only epilogue options at compile time (pre-activation save, aux / mask multiplies, atomic and
// strided fp32 stores, second fp32 output, column sums, scalar fallback); the host picks the variant per launch.
// v: accumulator + bias of columns [n0, n0 + 16) of this thread's row.  n0 is warp-uniform (column sums use the whole warp).
// SPLIT: out16 / out16p are fp16x3 pairs; the lo plane of each lies `lo16` elements after the hi plane.  The split variant is
// lean plus out32_id (the projector's vid_mem_proj output).
template <bool FULL, bool SPLIT>
__device__ __forceinline__ void epi_step(const GemmProblem& pr, const EpiRow& r, float (&v)[16], int n0, int fmt, int lane,
                                         long long lo16) {
  const int pN = pr.N;
  const int act = pr.act;
  const int ofmt = pr.out_fmt < 0 ? fmt : pr.out_fmt;
  const bool vec = FULL ? pr.vec_ok != 0 : true;  // the lean variant is only launched when every access can be vectorised
  const bool atomic = (pr.accumulate != 0) || (pr.ksplit > 1);
  const bool mask_mul = FULL && pr.mask_mul != 0;
  const float rsc = r.rsc;
  if (FULL && r.pre_row != nullptr && r.valid) {  // training: keep the pre-activation (needs N % 4 == 0, checked on the host)
    if (vec) {  // vec_ok implies N % 16 == 0: the whole step is in range
      st_global_256f(r.pre_row + n0, v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
      st_global_256f(r.pre_row + n0 + 8, v[8], v[9], v[10], v[11], v[12], v[13], v[14], v[15]);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (n0 + 4 * q < pN)
          *reinterpret_cast<float4*>(r.pre_row + n0 + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
  }
  if (FULL && act == ACT_GELU && r.dact_row != nullptr) {  // training forward: activation and its derivative in one pass
    uint32_t w8[8];  // the derivative, packed to 16 bits as it is formed (8 registers rather than 16 next to v)
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float g0, d0, g1, d1;
      gelu_erf_both(v[2 * q], g0, d0);
      gelu_erf_both(v[2 * q + 1], g1, d1);
      v[2 * q] = g0 * rsc;
      v[2 * q + 1] = g1 * rsc;
      w8[q] = cvt16x2(d0, d1, ofmt);
    }
    if (r.valid) {
      if (vec) {
        st_global_256(r.dact_row + n0, w8);
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (n0 + j < pN) r.dact_row[n0 + j] = (uint16_t)(w8[j / 2] >> (16 * (j & 1)));
      }
    }
  } else if (act == ACT_GELU) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = gelu_erf(v[j]) * rsc;
  } else if (act == ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f) * rsc;
  } else if (act == ACT_QUICKGELU) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = v[j] / (1.f + expf(-1.702f * v[j])) * rsc;
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] *= rsc;
  }
  if (vec) {
    if (r.valid) {
      if (r.resid_row != nullptr) {
        float rv[16];
        ld16f(r.resid_row + n0, rv);
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] += rv[j];
      }
      if (FULL && r.aux_row != nullptr) {
        float av[16];
        ld16f(r.aux_row + n0, av);
        if (pr.aux_mode == 1) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] *= gelu_erf_grad(av[j]);
        } else {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] *= av[j];
        }
      }
      if (FULL && r.mask_row != nullptr) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const uint4 mk = reinterpret_cast<const uint4*>(r.mask_row + n0)[q];
          const uint32_t w4[4] = {mk.x, mk.y, mk.z, mk.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (mask_mul) {  // saved activation derivative (GELU'): multiply
              v[8 * q + 2 * e] *= ld16((uint16_t)(w4[e] & 0xffff), fmt);
              v[8 * q + 2 * e + 1] *= ld16((uint16_t)(w4[e] >> 16), fmt);
            } else {  // ReLU mask: zero where the saved activation is <= 0
              if (!pos16((uint16_t)(w4[e] & 0xffff))) v[8 * q + 2 * e] = 0.f;
              if (!pos16((uint16_t)(w4[e] >> 16))) v[8 * q + 2 * e + 1] = 0.f;
            }
          }
        }
      }
      if (r.o32_row != nullptr) {
        if (FULL && atomic) {  // split-K / accumulate: 128-bit reductions (4x fewer L2 atomic operations than scalar REDs)
#pragma unroll
          for (int q = 0; q < 4; ++q)
            red_add_f32x4(r.o32_row + n0 + 4 * q, make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]));
        } else {
          st_global_256f(r.o32_row + n0, v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
          st_global_256f(r.o32_row + n0 + 8, v[8], v[9], v[10], v[11], v[12], v[13], v[14], v[15]);
        }
      }
      if ((FULL || SPLIT) && r.o32i_row != nullptr) {
        st_global_256f(r.o32i_row + n0, v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]);
        st_global_256f(r.o32i_row + n0 + 8, v[8], v[9], v[10], v[11], v[12], v[13], v[14], v[15]);
      }
      if (r.o16_row != nullptr) {
        uint32_t w8[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) w8[q] = cvt16x2(v[2 * q], v[2 * q + 1], ofmt);
        st_global_256(r.o16_row + n0, w8);
        if constexpr (SPLIT) {
#pragma unroll
          for (int q = 0; q < 8; ++q) w8[q] = cvt16x2_lo(v[2 * q], v[2 * q + 1]);
          st_global_256(r.o16_row + lo16 + n0, w8);
        }
      }
      if (r.o16p_row != nullptr) {
        float p[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) p[j] = v[j];
        if (r.add_row != nullptr) {
          float av[16];
          ld16f(r.add_row + n0, av);
#pragma unroll
          for (int j = 0; j < 16; ++j) p[j] += av[j];
        }
        uint32_t w8[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) w8[q] = cvt16x2(p[2 * q], p[2 * q + 1], ofmt);
        st_global_256(r.o16p_row + n0, w8);
        if constexpr (SPLIT) {
#pragma unroll
          for (int q = 0; q < 8; ++q) w8[q] = cvt16x2_lo(p[2 * q], p[2 * q + 1]);
          st_global_256(r.o16p_row + lo16 + n0, w8);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) v[j] = 0.f;  // invalid rows contribute nothing to the column sums
    }
  } else if constexpr (FULL) {
    // unaligned leading dimensions / ragged N (e.g. the [d, 2818] projector weight gradient, strided conv wgrad): scalar accesses
    const int cs32 = pr.cs32 > 1 ? pr.cs32 : 1;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n = n0 + j;
      float x = v[j];
      if (r.valid && n < pN) {
        if (r.resid_row != nullptr) x += r.resid_row[n];
        if (r.aux_row != nullptr) x *= (pr.aux_mode == 1) ? gelu_erf_grad(r.aux_row[n]) : r.aux_row[n];
        if (r.mask_row != nullptr) {
          if (mask_mul) x *= ld16(r.mask_row[n], fmt);
          else if (!pos16(r.mask_row[n])) x = 0.f;
        }
        if (r.o32_row != nullptr) {
          float* dst = r.o32_row + (size_t)n * cs32;
          if (atomic) atomicAdd(dst, x);
          else *dst = x;
        }
        if (r.o32i_row != nullptr) r.o32i_row[n] = x;
        if (r.o16_row != nullptr) {
          r.o16_row[n] = cvt16(x, ofmt);
          if constexpr (SPLIT) r.o16_row[lo16 + n] = cvt16_lo(x);
        }
        if (r.o16p_row != nullptr) {
          const float xp = x + (r.add_row ? r.add_row[n] : 0.f);
          r.o16p_row[n] = cvt16(xp, ofmt);
          if constexpr (SPLIT) r.o16p_row[lo16 + n] = cvt16_lo(xp);
        }
      } else {
        x = 0.f;
      }
      v[j] = x;
    }
  }
  if (FULL && pr.colsum != nullptr) {  // warp-uniform: column sums over this warp's 32 rows, one atomic per column
    const float sj = warp_colsum16(v, lane);  // 16 shuffles; lane l holds column l & 15
    if (lane < 16 && n0 + lane < pN) atomicAdd(pr.colsum + n0 + lane, sj * pr.colsum_scale);
  }
}

// ---- one consumer warpgroup: every tile of its schedule at tile width BN ----
// Each width has its own accumulator array, k-loops and epilogue read-out; the kernel picks the width once, before the first tile.
template <int CL, bool FULL, bool SPLIT, int BN>
__device__ __forceinline__ void consumer_tiles(const GemmGroup& g, Ring& ring, float* epi_buf, int crank, int cw, int lane) {
  using Cfg = GemmCfg<CL>;
  const int tid = threadIdx.x & 127;
  const int fr = 16 * (tid >> 5) + (lane >> 2);  // accumulator fragment: rows fr, fr + 8; columns 8 i + fc, + 1
  const int fc = 2 * (lane & 3);
  const int erow = tid & 63, ehalf = tid >> 6;  // epilogue: thread = row erow, columns [16 ehalf, +16) of each 32-column chunk
  float* ebuf = epi_buf + cw * 64 * Cfg::kEpiStride;
  const int fmt = g.fmt;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  TileInfo ti;
  bool first_tile = true;
  // the CTA's place in the deal is re-read from blockIdx / gridDim rather than kept in registers across the tile
  for (int rnd = 0; decode_tile<CL, SPLIT>(g, BN, gemm_deal_unit(gridDim.x / CL, blockIdx.x / CL, rnd), crank, ti); ++rnd) {
    const GemmProblem& pr = g.p[ti.p];
    const int bf = pr.a_fmt < 0 ? fmt : pr.a_fmt;  // both operands share it (checked on the host)
    if (first_tile && g.dbg != nullptr && ti.kb0 < ti.kb1) {
      mbar_wait(&ring.full[ring.stage], ring.phase);
      if (tid == 0 && cw == 0) stamp(g.dbg, 3);  // first operand stage landed
    }
    tile_mainloop_any<CL, SPLIT, BN>(acc, ring, bf, pr.a_mn, pr.b_mn, ti.kb0, ti.kb1, cw, tid, crank);
    if (tid == 0 && cw == 0) stamp(g.dbg, 4);  // last MMA of the tile retired
    first_tile = false;

    // ========================================= epilogue =========================================
    const int pM = pr.M, pN = pr.N, rps_in = pr.rps_in;
    const int m = ti.m_blk * GEMM_BM + cw * 64 + erow;
    int b = 0, l = m;
    if (rps_in > 0) {
      b = m / rps_in;
      l = m - b * rps_in;
    }
    const bool is_sep = (rps_in > 0) && (l == rps_in - 1);
    EpiRow r;
    r.valid = (m < pM) && !(pr.skip_sep && is_sep);
    r.rsc = pr.alpha;
    if (pr.row_scale != nullptr && m < pM) r.rsc *= pr.row_scale[b];
    if (pr.zero_sep && is_sep) r.rsc = 0.f;
    const size_t orow = (size_t)((rps_in > 0 ? b * pr.rps_out + l : m) + pr.row_off);
    r.resid_row = pr.resid ? pr.resid + orow * pr.ld_resid : nullptr;
    r.aux_row = (FULL && pr.aux32) ? pr.aux32 + orow * pr.ld_aux : nullptr;
    r.mask_row = (FULL && pr.mask16) ? pr.mask16 + orow * pr.ld_mask : nullptr;
    r.add_row = pr.addtab ? pr.addtab + (size_t)m * pr.ld_addtab : nullptr;
    r.o32_row = pr.out32 ? pr.out32 + orow * pr.ld32 : nullptr;
    r.o32i_row = ((FULL || SPLIT) && pr.out32_id) ? pr.out32_id + (size_t)m * pr.ld32_id : nullptr;
    r.o16_row = pr.out16 ? pr.out16 + orow * pr.ld16 : nullptr;
    r.o16p_row = pr.out16p ? pr.out16p + orow * pr.ld16 : nullptr;
    r.pre_row = (FULL && pr.pre32) ? pr.pre32 + orow * pr.ld_pre : nullptr;
    r.dact_row = (FULL && pr.dact16) ? pr.dact16 + orow * pr.ld_dact : nullptr;
    const float* __restrict__ bias = (ti.split == 0) ? pr.bias : nullptr;
    const int nt0 = ti.n_blk * BN;
    // 32-column chunks; when BN % 32 == 16 the last chunk holds 16 columns (its ehalf = 1 half is neither staged nor read).
    // The chunk loop stays rolled so that each width carries one copy of the epilogue; only the staging of a chunk's
    // accumulators (registers named at compile time) is unrolled.
#pragma unroll 1
    for (int cc = 0; cc < (BN + 31) / 32 && nt0 + cc * 32 < pN; ++cc) {  // warpgroup-uniform
#pragma unroll
      for (int c = 0; c < (BN + 31) / 32; ++c) {
        if (c == cc) {
#pragma unroll
          for (int ii = 0; ii < 4; ++ii) {
            const int i = 4 * c + ii;
            if (8 * i < BN) {
              *reinterpret_cast<float2*>(ebuf + fr * Cfg::kEpiStride + 8 * ii + fc) = make_float2(acc[4 * i], acc[4 * i + 1]);
              *reinterpret_cast<float2*>(ebuf + (fr + 8) * Cfg::kEpiStride + 8 * ii + fc) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
            }
          }
        }
      }
      named_bar_sync(1 + cw, 128);
      const int n0 = nt0 + cc * 32 + ehalf * 16;
      if (cc * 32 + ehalf * 16 < BN && n0 < pN) {  // warp-uniform (a warp's rows share ehalf)
        float v[16];
        ld16f(ebuf + erow * Cfg::kEpiStride + ehalf * 16, v);
        if (bias != nullptr) {
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] += (n0 + j < pN) ? __ldg(bias + n0 + j) : 0.f;
        }
        epi_step<FULL, SPLIT>(pr, r, v, n0, fmt, lane, g.lo16);
      }
      named_bar_sync(1 + cw, 128);
    }
    // epilogue of the tile done (second warpgroup's first thread; threadIdx.x is read again rather than a predicate kept
    // across the tile, which keeps the FULL variant free of spills)
    if (threadIdx.x == 128) stamp(g.dbg, 6);
  }
}

// SPLIT (fp16x3, CL = 1, K-major operands only): tm_a / tm_b are 3-D maps whose third coordinate selects the hi (0) or lo (1)
// plane.  A problem walks its taps x kblk_per_tap k-blocks three times - (A hi, B hi), (A lo, B hi), (A hi, B lo) - into the
// same accumulators; only the producer knows about the planes.
template <int CL, bool FULL, bool SPLIT = false>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_wgmma_kernel(const __grid_constant__ GemmGroup g) {
  using Cfg = GemmCfg<CL>;
  const int BN = g.bn;
  const int kStageBytes = Cfg::stage_bytes(BN);
  const int kStages = Cfg::num_stages(BN);
  const int crank = (CL > 1) ? (int)cluster_ctarank() : 0;  // rank inside the cluster
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t align_off = (1024u - (raw_addr & 1023u)) & 1023u;  // 0 when the runtime honours the 1024 B alignment
  uint8_t* smem = smem_raw + align_off;

  uint8_t* stage_base = smem;
  float* epi_buf = reinterpret_cast<float*>(smem + Cfg::kRingBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(epi_buf + Cfg::kEpiFloats);
  uint64_t* full_bar = bars;                     // [kMaxStages]
  uint64_t* empty_bar = bars + Cfg::kMaxStages;  // [kMaxStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) stamp(g.dbg, 0);  // kernel entry (profiling buffer only; never an output of a preceding kernel)

  if (warp == 8 && lane == 0) {
    for (int p = 0; p < g.num; ++p) {
      tma_prefetch_desc(&g.p[p].tm_a);
      tma_prefetch_desc(&g.p[p].tm_b);
    }
  }
  if (warp == 0 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * CL);  // both consumer warpgroups of every CTA the stage's B tile is multicast to
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();  // the peer's barriers are initialised before any multicast can reach them
  pdl_launch_dependents();
  pdl_wait();  // barriers and tensor-map prefetch happened under the previous kernel's tail; its results are visible from here
  if (threadIdx.x == 0) stamp(g.dbg, 1);  // setup done

  if (wg == 2) {
    setmaxnreg_dec<40>();
    if (warp == 8) {
      // ======================================= TMA producer =======================================
      // The whole warp walks the schedule convergently and ONE elected lane issues (elect.sync), so that the TMA operands are
      // provably warp-uniform.
      int stage = 0;
      uint32_t phase = 0;
      TileInfo ti;
      for (int r = 0; decode_tile<CL, SPLIT>(g, BN, gemm_deal_unit(gridDim.x / CL, blockIdx.x / CL, r), crank, ti); ++r) {
        const GemmProblem& pr = g.p[ti.p];
        const int m0 = ti.m_blk * GEMM_BM;
        const int n0 = ti.n_blk * BN;
        for (int kb = ti.kb0; kb < ti.kb1; ++kb) {
          int kbt = kb, plane_a = 0, plane_b = 0;
          if constexpr (SPLIT) {
            const int per_product = pr.taps * pr.kblk_per_tap;
            const int prod = kb / per_product;  // 0: hi x hi, 1: lo x hi, 2: hi x lo
            kbt = kb - prod * per_product;
            plane_a = prod == 1;
            plane_b = prod == 2;
          }
          const int tap = kbt / pr.kblk_per_tap;
          const int kk = (kbt - tap * pr.kblk_per_tap) * GEMM_BK;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = stage_base + stage * kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          const int a0 = pr.ca.base0 + m0 * pr.ca.mn0s + tap * pr.ca.tap0 + kk * pr.ca.k0s;
          const int a1 = pr.ca.base1 + m0 * pr.ca.mn1s + tap * pr.ca.tap1 + kk * pr.ca.k1s;
          const int b0 = pr.cb.base0 + n0 * pr.cb.mn0s + tap * pr.cb.tap0 + kk * pr.cb.k0s;
          const int b1 = pr.cb.base1 + n0 * pr.cb.mn1s + tap * pr.cb.tap1 + kk * pr.cb.k1s;
          if (elect_one()) {
            mbar_arrive_expect_tx(&full_bar[stage], Cfg::kABytes + BN * 128);
            if constexpr (SPLIT) {
              tma_load_3d(sa, &pr.tm_a, &full_bar[stage], a0, a1, plane_a);
              tma_load_3d(sb, &pr.tm_b, &full_bar[stage], b0, b1, plane_b);
            } else if (!pr.a_mn) {
              tma_load_2d(sa, &pr.tm_a, &full_bar[stage], a0, a1);
            } else {
#pragma unroll
              for (int j = 0; j < GEMM_BM / 64; ++j) tma_load_2d(sa + j * 8192, &pr.tm_a, &full_bar[stage], a0 + 64 * j, a1);
            }
            if constexpr (SPLIT) {
            } else if (CL == 1) {
              if (!pr.b_mn) {
                tma_load_2d(sb, &pr.tm_b, &full_bar[stage], b0, b1);
              } else if (pr.b_3d) {
                tma_load_3d(sb, &pr.tm_b, &full_bar[stage], 0, b1, b0 >> 6);  // all BN/64 blocks of the k-block in one TMA operation
              } else {
                for (int j = 0; j < BN / 64; ++j) tma_load_2d(sb + j * 8192, &pr.tm_b, &full_bar[stage], b0 + 64 * j, b1);
              }
            } else {
              const int hr = BN / 2;  // tensor-map box = BN/2 rows: this CTA's half of the B tile, multicast to both CTAs
              tma_load_2d_mc(sb + crank * hr * 128, &pr.tm_b, &full_bar[stage], b0, b1 + crank * hr, (uint16_t)0x3);
            }
          }
          __syncwarp();
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
      if (lane == 0) stamp(g.dbg, 2);  // all TMA loads issued
    }
  } else {
    setmaxnreg_inc<232>();
    // ======================================= consumers =======================================
    // warpgroup wg computes rows [64 wg, 64 wg + 64) of each tile.  The host accepts multiples of 16 in [32, 256] (of 32 in
    // clusters), so only those widths are compiled.
    Ring ring{stage_base, full_bar, empty_bar, kStageBytes, kStages, 0, 0u};
    switch (BN >> 4) {
#define UV_BN_CASE(k) \
  case k: consumer_tiles<CL, FULL, SPLIT, 16 * k>(g, ring, epi_buf, crank, wg, lane); break;
#define UV_BN_CASE_ODD(k) \
  case k: if constexpr (CL == 1) consumer_tiles<CL, FULL, SPLIT, 16 * k>(g, ring, epi_buf, crank, wg, lane); break;
      UV_BN_CASE(2) UV_BN_CASE_ODD(3) UV_BN_CASE(4) UV_BN_CASE_ODD(5) UV_BN_CASE(6) UV_BN_CASE_ODD(7) UV_BN_CASE(8)
      UV_BN_CASE_ODD(9) UV_BN_CASE(10) UV_BN_CASE_ODD(11) UV_BN_CASE(12) UV_BN_CASE_ODD(13) UV_BN_CASE(14) UV_BN_CASE_ODD(15)
      UV_BN_CASE(16)
#undef UV_BN_CASE_ODD
#undef UV_BN_CASE
      default: __trap();  // launch_gemm_group rejects every other width; without consumers the producer would wait forever
    }
  }

  __syncthreads();
  if (CL > 1) cluster_sync_all();  // no CTA leaves while its peer may still multicast into it or signal its barriers
  if (threadIdx.x == 0) stamp(g.dbg, 7);  // exit
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static unsigned long long* g_timeline = nullptr;
void set_gemm_timeline_buffer(unsigned long long* buf) { g_timeline = buf; }
bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("UNIVTG_PDL");
    on = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return on == 1;
}
long long* launch_counter() {
  static long long n = 0;
  return &n;
}
static thread_local char g_err[512] = "";
const char* last_error() { return g_err; }
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || p == nullptr) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (cudaError %d)", (int)e);
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// Tensor maps are pure functions of (base, extents, pitch, box): the training path describes ~250 operand views per step and, with
// pooled workspaces, describes the SAME views every step - a small direct-mapped cache turns ~250 driver calls per step
// (cuTensorMapEncodeTiled, ~1.5 us each on the host) into hash look-ups.  Thread-local: one process per GPU, one host thread.
struct TmapKey {
  const void* base;
  uint64_t rows, cols, ld;
  uint32_t box_rows, box_cols, kind;
  uint64_t plane;  // kind 4 (fp16x3 pair): element offset of the lo plane
  bool operator==(const TmapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && box_cols == o.box_cols && kind == o.kind &&
           plane == o.plane;
  }
};
struct TmapSlot {
  TmapKey key;
  CUtensorMap map;
  bool used;
};
constexpr int kTmapCacheSlots = 4096;
static thread_local TmapSlot* g_tmap_cache = nullptr;
static inline TmapSlot* tmap_slot(const TmapKey& k) {
  if (g_tmap_cache == nullptr) g_tmap_cache = static_cast<TmapSlot*>(calloc(kTmapCacheSlots, sizeof(TmapSlot)));
  uint64_t h = reinterpret_cast<uintptr_t>(k.base) * 0x9E3779B97F4A7C15ull;
  h ^= (k.rows * 0xC2B2AE3D27D4EB4Full) ^ (k.cols << 17) ^ (k.ld << 29) ^ ((uint64_t)k.box_rows << 41) ^ ((uint64_t)k.box_cols << 47) ^ ((uint64_t)k.kind << 55);
  h ^= k.plane * 0x94D049BB133111EBull;
  h ^= h >> 29;
  return g_tmap_cache ? &g_tmap_cache[h & (kTmapCacheSlots - 1)] : nullptr;
}

// The tensor map of `key` from the cache, or encoded over 16-bit elements (128-byte swizzle, zero fill out of bounds) and stored.
// dims / box: innermost first; strides: bytes between consecutive entries of dims 1 .. rank - 1.
static int make_tmap_cached(CUtensorMap* out, const TmapKey& key, cuuint32_t rank, const cuuint64_t* dims, const cuuint64_t* strides,
                            const cuuint32_t* box) {
  TmapSlot* slot = tmap_slot(key);
  if (slot != nullptr && slot->used && slot->key == key) {
    *out = slot->map;
    return 0;
  }
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return 1;
  const char* what = key.kind == 4 ? "fp16x3 pair" : key.kind == 3 ? "3-D MN-major B" : "2-D";
  bool aligned = (reinterpret_cast<uintptr_t>(key.base) & 15) == 0;
  for (cuuint32_t i = 0; i + 1 < rank; ++i) aligned = aligned && strides[i] % 16 == 0;
  if (!aligned) {
    set_error("tensor map (%s): base %p, pitch %llu B and lo-plane offset %llu B must be 16-byte aligned", what, key.base,
              (unsigned long long)(key.ld * 2), (unsigned long long)(key.plane * 2));
    return 2;
  }
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT16, rank, const_cast<void*>(key.base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (%s) failed: CUresult %d (rows %llu cols %llu ld %llu lo %llu box %ux%u)", what, (int)r,
              (unsigned long long)key.rows, (unsigned long long)key.cols, (unsigned long long)key.ld, (unsigned long long)key.plane,
              key.box_rows, key.box_cols);
    return 3;
  }
  if (slot != nullptr) {
    slot->key = key;
    slot->map = *out;
    slot->used = true;
  }
  return 0;
}

int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                 uint32_t box_cols) {
  const cuuint64_t dims[2] = {cols, rows}, strides[1] = {ld_elems * 2};
  const cuuint32_t box[2] = {box_cols, box_rows};
  return make_tmap_cached(out, TmapKey{base, rows, cols, ld_elems, box_rows, box_cols, 2u, 0}, 2, dims, strides, box);
}

int make_tmap_split(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                    uint32_t box_cols, uint64_t lo_elems) {
  const cuuint64_t dims[3] = {cols, rows, 2}, strides[2] = {ld_elems * 2, lo_elems * 2};
  const cuuint32_t box[3] = {box_cols, box_rows, 1};
  return make_tmap_cached(out, TmapKey{base, rows, cols, ld_elems, box_rows, box_cols, 4u, lo_elems}, 3, dims, strides, box);
}

int make_tmap_b_mn(GemmProblem& p, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, int bn) {
  p.b_3d = 0;
  if (cols % 64 != 0 || bn % 64 != 0 || bn < 64) return make_tmap_2d(&p.tm_b, base, rows, cols, ld_elems, 64, 64);
  const cuuint64_t dims[3] = {64, rows, cols / 64}, strides[2] = {ld_elems * 2, 128};
  const cuuint32_t box[3] = {64, 64, (cuuint32_t)(bn / 64)};
  const int rc = make_tmap_cached(&p.tm_b, TmapKey{base, rows, cols, ld_elems, (uint32_t)bn, 64u, 3u, 0}, 3, dims, strides, box);
  if (rc == 0) p.b_3d = bn / 64;
  return rc;
}

int launch_gemm_group(GemmGroup& g, int bn, int num_sms, cudaStream_t stream, int* used_full) {
  using Cfg = GemmCfg<1>;
  static_assert(GemmCfg<1>::kSmemBytes == GemmCfg<2>::kSmemBytes, "both variants use the same dynamic shared memory size");
  if (g.num < 1 || g.num > GEMM_MAX_GROUP) {
    set_error("gemm group size %d out of range", g.num);
    return (int)cudaErrorInvalidValue;
  }
  if (bn < 32 || bn > 256 || bn % 16 != 0) {
    set_error("unsupported BN %d (multiple of 16 in [32, 256])", bn);
    return (int)cudaErrorInvalidValue;
  }
  const int cl = g.cluster == 2 ? 2 : 1;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_wgmma_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_wgmma_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_wgmma_kernel<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(gemm_wgmma_kernel<1, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(gemm, smem=%d): %s", Cfg::kSmemBytes, cudaGetErrorString(e));
      return (int)e;
    }
    attr_set = true;
  }
  if (cl == 2 && (bn % 32 != 0)) {
    set_error("cluster GEMM needs BN %% 32 == 0 (got %d)", bn);
    return (int)cudaErrorInvalidValue;
  }
  if (g.split && (cl != 1 || g.fmt != 0)) {
    set_error("fp16x3 gemm group: needs cluster 1 and group format 0 (got cluster %d, fmt %d)", cl, g.fmt);
    return (int)cudaErrorInvalidValue;
  }
  int total = 0;
  for (int p = 0; p < g.num; ++p) {
    const GemmProblem& pr = g.p[p];
    if (g.split && (pr.a_mn || pr.b_mn || pr.a_fmt > 0 || pr.b_fmt > 0 || pr.out_fmt > 0)) {
      set_error("gemm problem %d: fp16x3 problems need K-major fp16 operands and output", p);
      return (int)cudaErrorInvalidValue;
    }
    if (pr.ksplit < 1 || pr.taps < 1 || pr.kblk_per_tap < 1 || pr.ksplit > pr.taps * pr.kblk_per_tap * (g.split ? 3 : 1)) {
      set_error("gemm problem %d: bad k configuration (taps %d kblk %d ksplit %d)", p, pr.taps, pr.kblk_per_tap, pr.ksplit);
      return (int)cudaErrorInvalidValue;
    }
    if (!pr.b_mn && pr.b_box_rows != bn / cl) {
      set_error("gemm problem %d: B tensor-map box has %d rows but the launch uses bn %d (cluster %d)", p, pr.b_box_rows, bn, cl);
      return (int)cudaErrorInvalidValue;
    }
    if (cl == 2 && pr.b_mn) {
      set_error("gemm problem %d: cluster launches need a K-major B operand", p);
      return (int)cudaErrorInvalidValue;
    }
    if (pr.b_mn && pr.b_3d != 0 && pr.b_3d != bn / 64) {
      set_error("gemm problem %d: 3-D B tensor map was built for bn %d (got bn %d)", p, 64 * pr.b_3d, bn);
      return (int)cudaErrorInvalidValue;
    }
    if (pr.b_mn && bn % (64 * cl) != 0) {
      set_error("gemm problem %d: MN-major B needs BN %% %d == 0 (got %d)", p, 64 * cl, bn);
      return (int)cudaErrorInvalidValue;
    }
    // split-K tiles and `accumulate` add partial sums into out32: only options that are linear in the accumulator (bias is added by
    // split 0 alone) may run on a partial sum; an activation, a residual or a 16-bit / identity-row store of one would be wrong
    if (pr.ksplit > 1 || pr.accumulate) {
      const char* bad = pr.dact16 ? "dact16" : pr.act != ACT_NONE ? "act" : pr.resid ? "resid" : pr.out16 ? "out16"
                        : pr.out16p ? "out16p" : pr.out32_id ? "out32_id" : nullptr;
      if (bad != nullptr) {
        set_error("gemm problem %d: %s cannot be combined with %s (each split would apply it to a partial sum)", p, bad,
                  pr.ksplit > 1 ? "ksplit > 1" : "accumulate");
        return (int)cudaErrorInvalidValue;
      }
    }
    const int fa = pr.a_fmt < 0 ? g.fmt : pr.a_fmt, fb = pr.b_fmt < 0 ? g.fmt : pr.b_fmt;
    if (fa != fb) {
      set_error("gemm problem %d: A and B must share one 16-bit format (wgmma), got %d and %d", p, fa, fb);
      return (int)cudaErrorInvalidValue;
    }
    const int total_kb = pr.taps * pr.kblk_per_tap * (g.split ? 3 : 1);
    const int per = (total_kb + pr.ksplit - 1) / pr.ksplit;
    if ((pr.ksplit - 1) * per >= total_kb) {
      set_error("gemm problem %d: ksplit %d leaves an empty split for %d k-blocks", p, pr.ksplit, total_kb);
      return (int)cudaErrorInvalidValue;
    }
    total += ((((pr.M + GEMM_BM - 1) / GEMM_BM) + cl - 1) / cl) * ((pr.N + bn - 1) / bn) * pr.ksplit;  // tiles (CL=1) or tile pairs
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    GemmProblem& w = g.p[p];
    // epilogue (thread = row, 16 columns per step): 128-bit accesses need N % 16 == 0 and aligned leading dimensions
    w.vec_ok = (pr.N % 16 == 0) && (pr.cs32 <= 1) && (!pr.aux32 || (al16(pr.aux32) && pr.ld_aux % 4 == 0)) &&
               (!pr.pre32 || (al16(pr.pre32) && pr.ld_pre % 4 == 0)) && (!pr.dact16 || (al16(pr.dact16) && pr.ld_dact % 8 == 0)) && (!pr.mask16 || (al16(pr.mask16) && pr.ld_mask % 8 == 0)) &&
               (!pr.resid || (al16(pr.resid) && pr.ld_resid % 4 == 0)) && (!pr.addtab || (al16(pr.addtab) && pr.ld_addtab % 4 == 0)) &&
               (!pr.out32 || (al16(pr.out32) && pr.ld32 % 4 == 0)) && (!pr.out32_id || (al16(pr.out32_id) && pr.ld32_id % 4 == 0)) &&
               ((!pr.out16 && !pr.out16p) || (pr.ld16 % 8 == 0 && al16(pr.out16) && al16(pr.out16p) && g.lo16 % 8 == 0));
    auto al32 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 31) == 0; };
    // 256-bit accesses (one whole 32-byte sector per thread and instruction) when every leading dimension keeps rows 32-byte aligned
    if (w.vec_ok && (!pr.pre32 || (al32(pr.pre32) && pr.ld_pre % 8 == 0)) && (!pr.dact16 || (al32(pr.dact16) && pr.ld_dact % 16 == 0)) && (!pr.aux32 || (al32(pr.aux32) && pr.ld_aux % 8 == 0)) && (!pr.addtab || (al32(pr.addtab) && pr.ld_addtab % 8 == 0)) && (!pr.resid || (al32(pr.resid) && pr.ld_resid % 8 == 0)) &&
        (!pr.out32 || (al32(pr.out32) && pr.ld32 % 8 == 0)) && (!pr.out32_id || (al32(pr.out32_id) && pr.ld32_id % 8 == 0)) &&
        ((!pr.out16 && !pr.out16p) || (pr.ld16 % 16 == 0 && al32(pr.out16) && al32(pr.out16p) && g.lo16 % 16 == 0)))
      w.vec_ok = 2;
  }
  if (total == 0) return 0;
  bool full = false;  // does any problem of the group need an epilogue option only the FULL variant compiles in?
  for (int p = 0; p < g.num; ++p) {
    const GemmProblem& pr = g.p[p];
    full = full || pr.vec_ok != 2 || pr.pre32 || pr.dact16 || pr.aux32 || pr.mask16 || pr.accumulate || pr.ksplit > 1 ||
           (pr.out32_id && !g.split) || pr.colsum || pr.cs32 > 1;  // the split lean variant also stores out32_id
  }
  if (g.split && full) {  // inference products only: the lean epilogue (the FULL one would spill with the split producer)
    set_error("fp16x3 gemm group: needs the lean epilogue (N %% 16 == 0, 32-byte aligned outputs and lo planes, no training options or split-K)");
    return (int)cudaErrorInvalidValue;
  }
  if (used_full) *used_full = full ? 1 : 0;
  g.bn = bn;
  g.dbg = g_timeline;
  GemmGroup gl = g;  // the launched copy, problems in deal order (the caller's order stays as it was)
  gemm_deal_order(gl, nullptr);
  cudaError_t e;
  if (cl == 1) {
    const int grid = total < num_sms ? total : num_sms;
    if (g.split) {
      launch_k(gemm_wgmma_kernel<1, false, true>, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, gl);
    } else if (full) {
      launch_k(gemm_wgmma_kernel<1, true>, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, gl);
    } else {
      launch_k(gemm_wgmma_kernel<1, false>, dim3(grid), dim3(kGemmThreads), Cfg::kSmemBytes, stream, gl);
    }
    e = cudaGetLastError();
  } else {
    const int max_clusters = num_sms / 2;
    const int clusters = total < max_clusters ? total : max_clusters;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(2 * clusters);
    cfg.blockDim = dim3(kGemmThreads);
    cfg.dynamicSmemBytes = Cfg::kSmemBytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
    ++*launch_counter();
    e = full ? cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<2, true>, gl) : cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<2, false>, gl);
  }
  if (e != cudaSuccess) {
    set_error("gemm launch failed: %s", cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

void gemm_deal_order(GemmGroup& g, int* perm) {
  const bool split = g.split != 0;
  int order[GEMM_MAX_GROUP];
  for (int p = 0; p < g.num; ++p) {  // stable insertion: equal units keep the problem order
    const int kb = gemm_unit_kblocks(g.p[p], split);
    int i = p;
    for (; i > 0 && gemm_unit_kblocks(g.p[order[i - 1]], split) < kb; --i) order[i] = order[i - 1];
    order[i] = p;
  }
  GemmProblem sorted[GEMM_MAX_GROUP];
  for (int i = 0; i < g.num; ++i) sorted[i] = g.p[order[i]];
  for (int i = 0; i < g.num; ++i) {
    g.p[i] = sorted[i];
    if (perm) perm[i] = order[i];
  }
}

// The scheduling fields of a launch of problems M x N x (kblocks 64-wide k-blocks), split ks ways (CL = 1, plain taps).
static void deal_group(GemmGroup& g, const int* Ms, const int* Ns, const int* kblocks, const int* ks, int num, int* perm = nullptr) {
  memset(&g, 0, sizeof(g));
  g.num = num;
  for (int p = 0; p < num; ++p) {
    g.p[p].M = Ms[p];
    g.p[p].N = Ns[p];
    g.p[p].taps = 1;
    g.p[p].kblk_per_tap = kblocks[p];
    g.p[p].ksplit = ks[p];
  }
  gemm_deal_order(g, perm);
}

static int deal_units(const GemmGroup& g, int bn) {
  int total = 0;
  for (int p = 0; p < g.num; ++p) total += ((g.p[p].M + GEMM_BM - 1) / GEMM_BM) * ((g.p[p].N + bn - 1) / bn) * g.p[p].ksplit;
  return total;
}

int gemm_deal_ctas(const int* Ms, const int* Ns, const int* kblocks, const int* ksplit, int num, int num_sms, int bn, int* cta, int cap) {
  if (num < 1 || num > GEMM_MAX_GROUP || num_sms < 1 || bn < 16) return -1;
  for (int p = 0; p < num; ++p)
    if (Ms[p] < 1 || Ns[p] < 1 || kblocks[p] < 1 || ksplit[p] < 1 || ksplit[p] > kblocks[p]) return -1;
  GemmGroup g;
  int perm[GEMM_MAX_GROUP];  // deal position -> problem
  deal_group(g, Ms, Ns, kblocks, ksplit, num, perm);
  const int total = deal_units(g, bn);
  int first[GEMM_MAX_GROUP];  // index of problem p's first unit in `cta` (problem order)
  for (int p = 0, u = 0; p < num; ++p) {
    first[p] = u;
    u += ((Ms[p] + GEMM_BM - 1) / GEMM_BM) * ((Ns[p] + bn - 1) / bn) * ksplit[p];
  }
  for (int u = 0; u < total && u < cap; ++u) cta[u] = -1;
  const int n = total < num_sms ? total : num_sms;  // the grid launch_gemm_group runs
  for (int c = 0; c < n; ++c) {
    TileInfo ti;
    for (int r = 0; decode_tile<1, false>(g, bn, gemm_deal_unit(n, c, r), 0, ti); ++r) {
      const int p = perm[ti.p];
      const int tm = (Ms[p] + GEMM_BM - 1) / GEMM_BM, tn = (Ns[p] + bn - 1) / bn;
      const int u = first[p] + (ti.split * tm + ti.m_blk) * tn + ti.n_blk;
      if (u < cap) cta[u] = cta[u] == -1 ? c : -2;
    }
  }
  return total;
}

// Modelled time (us) of one launch: the busiest CTA of the deal that the kernel runs.  The constants are a model, not a
// measurement: a 64-wide k-block of a 128 x bn tile is 128 * bn * 64 multiply-adds at the data-sheet dense fp16 rate of one SM
// (989 TFLOP/s over 132 SMs, ~0.0018 us per tile column) plus ~0.15 us of TMA / barrier overhead, ~1 us from kernel entry to
// the first MMA, and per unit an epilogue of ~0.5 us + 2 us x bn/256 (3 us x bn/256 for a split-K unit, which reduces into its
// output), of which only a fraction is exposed when the CTA has further units to run.
static double model_launch_us(const GemmGroup& g, int bn, int num_sms) {
  const int total = deal_units(g, bn);
  const int n = total < num_sms ? total : num_sms;
  const double kb_us = 0.15 + 0.0018 * bn;
  double worst = 0.0;
  for (int c = 0; c < n; ++c) {
    double busy = 0.0, last_epi = 0.0;
    TileInfo ti;
    for (int r = 0; decode_tile<1, false>(g, bn, gemm_deal_unit(n, c, r), 0, ti); ++r) {
      last_epi = 0.5 + bn * (g.p[ti.p].ksplit > 1 ? 3.0 : 2.0) / 256.0;
      busy += kb_us * (double)(ti.kb1 - ti.kb0) + 0.3 * last_epi;
    }
    busy += 0.7 * last_epi;
    worst = busy > worst ? busy : worst;
  }
  return 1.0 + worst;
}

// Every combination of per-problem split factors (powers of two up to max_split[p], at least 4 k-blocks per split) at every
// width; ties keep the smaller splits and the wider tile.  The plan asks the same questions every step: a small cache of
// answers keeps the search off the host's launch path.
struct TileQuery {
  int Ms[GEMM_MAX_GROUP], Ns[GEMM_MAX_GROUP], kb[GEMM_MAX_GROUP], max_split[GEMM_MAX_GROUP];
  int num, num_sms, step;
};
TileChoice choose_tile(const int* Ms, const int* Ns, const int* kblocks, const int* max_split, int num, int num_sms, int step) {
  TileQuery q;
  memset(&q, 0, sizeof(q));
  for (int p = 0; p < num; ++p) {
    q.Ms[p] = Ms[p];
    q.Ns[p] = Ns[p];
    q.kb[p] = kblocks[p];
    q.max_split[p] = max_split[p];
  }
  q.num = num;
  q.num_sms = num_sms;
  q.step = step;
  constexpr int kCache = 32;
  static thread_local TileQuery cq[kCache];
  static thread_local TileChoice ca[kCache];
  static thread_local int cn = 0;
  for (int i = 0; i < cn && i < kCache; ++i)
    if (memcmp(&cq[i], &q, sizeof(q)) == 0) return ca[i];

  TileChoice best;
  memset(&best, 0, sizeof(best));
  double best_t = -1.0;
  int ks[GEMM_MAX_GROUP];
  for (int p = 0; p < num; ++p) ks[p] = 1;
  GemmGroup g;
  for (;;) {
    deal_group(g, Ms, Ns, kblocks, ks, num);
    for (int bn = 256; bn >= 64; bn -= step) {
      const double t = model_launch_us(g, bn, num_sms);
      if (best_t < 0 || t < best_t - 1e-9) {
        best_t = t;
        best.bn = bn;
        best.ksplit = 1;
        for (int p = 0; p < GEMM_MAX_GROUP; ++p) {
          best.ks[p] = p < num ? ks[p] : 1;
          best.ksplit = best.ks[p] > best.ksplit ? best.ks[p] : best.ksplit;
        }
      }
    }
    int p = 0;  // next combination (mixed radix, problem 0 fastest)
    for (; p < num; ++p) {
      if (ks[p] * 2 <= max_split[p] && ks[p] * 2 * 4 <= kblocks[p]) {
        ks[p] *= 2;
        break;
      }
      ks[p] = 1;
    }
    if (p == num) break;
  }
  cq[cn % kCache] = q;
  ca[cn % kCache] = best;
  ++cn;
  return best;
}

}  // namespace uv
