// Bandwidth-bound row kernels of the UniVTG hot path (HBM roofline; 128-bit coalesced accesses, warp reductions):
//   * layernorm_rows     - nn.LayerNorm (eps 1e-5, biased variance) of LinearLayer (model/univtg.py:392,401) and of
//                          norm1/norm2 (model/transformer_encoder_droppath.py:99-100,121,125); emits the fp32 residual
//                          stream plus the 16-bit GEMM operands x and x+pos (q = k = x + pos, :117).
//   * sine_pos_table     - PositionEmbeddingSine.forward (model/position_encoding.py:60-83)
//   * pool_saliency      - WeightedPool.forward (model/univtg.py:43-49) + cosine saliency (:146-147)
//   * conv_head_final    - third Conv1d (k=3) of class_embed / span_embed + sigmoid + (-1,+1) sign (model/univtg.py:129-136)
#include <math.h>

#include "kernels.h"
#include "ptx.cuh"
#include "rowops.h"

namespace uv {

// ------------------------------------------------------------------------------------------------
// LayerNorm over rows.  One warp per row.
// TXT: the text rows of out16p also get a.pos_txt (learned text positions); a separate instantiation, so the kernels without
// text positions are compiled exactly as before.
// SPLIT: fp16x3 (LnArgs.split) - add16 is read and out16 / out16p / outc are written as hi / lo pairs, the lo plane `a.lo`
// elements after the hi plane; again a separate instantiation.
// ------------------------------------------------------------------------------------------------
template <bool TXT = false, bool SPLIT = false>
struct LnStore {
  const LnArgs& a;
  const unsigned long long seed;  // a.drop's seed, resolved once per row (drop_seed); only the seed is held, not a spec copy
  int row, b, l;
  bool has_pos;
  size_t prow, crow, trow;
  __device__ LnStore(const LnArgs& a_, int row_) : a(a_), seed(a_.drop.on ? drop_seed(a_.drop) : 0ull), row(row_) {
    b = 0;
    l = row;
    if (a.L > 0) {
      b = row / a.L;
      l = row - b * a.L;
    }
    has_pos = (a.pos != nullptr) && (a.L > 0) && (l < a.Lv);
    prow = (size_t)b * a.Lv + l;
    crow = (size_t)1 + (size_t)b * (a.Lv + 1) + l;
    trow = (size_t)b * (a.L - a.Lv) + (l - a.Lv);
  }
  __device__ __forceinline__ void store4(int j, float4 v) const {
    if (a.out32) *reinterpret_cast<float4*>(a.out32 + (size_t)row * a.d + j) = v;
    if (a.mul32) {
      const float4 m = *reinterpret_cast<const float4*>(a.mul32 + (size_t)row * a.d + j);
      v.x *= m.x; v.y *= m.y; v.z *= m.z; v.w *= m.w;
    } else if (a.drop.on) {
      const float4 m = drop_mul4(drop_with_seed(a.drop, seed), (unsigned int)row, (unsigned int)j);
      v.x *= m.x; v.y *= m.y; v.z *= m.z; v.w *= m.w;
    }
    uint2 pk, pkl = make_uint2(0u, 0u);
    pk.x = cvt16x2(v.x, v.y, a.fmt);
    pk.y = cvt16x2(v.z, v.w, a.fmt);
    if constexpr (SPLIT) pkl = make_uint2(cvt16x2_lo(v.x, v.y), cvt16x2_lo(v.z, v.w));
    if (a.out16) {
      *reinterpret_cast<uint2*>(a.out16 + (size_t)row * a.ld16 + j) = pk;
      if constexpr (SPLIT) *reinterpret_cast<uint2*>(a.out16 + a.lo + (size_t)row * a.ld16 + j) = pkl;
    }
    if (a.out16p) {
      uint2 pp = pk, ppl = pkl;
      if (has_pos) {
        const float4 p = *reinterpret_cast<const float4*>(a.pos + prow * a.d + j);
        pp.x = cvt16x2(v.x + p.x, v.y + p.y, a.fmt);
        pp.y = cvt16x2(v.z + p.z, v.w + p.w, a.fmt);
        if constexpr (SPLIT) ppl = make_uint2(cvt16x2_lo(v.x + p.x, v.y + p.y), cvt16x2_lo(v.z + p.z, v.w + p.w));
      }
      if constexpr (TXT) {
        if (a.L > 0 && l >= a.Lv) {
          const float4 p = *reinterpret_cast<const float4*>(a.pos_txt + trow * a.d + j);
          pp.x = cvt16x2(v.x + p.x, v.y + p.y, a.fmt);
          pp.y = cvt16x2(v.z + p.z, v.w + p.w, a.fmt);
          if constexpr (SPLIT) ppl = make_uint2(cvt16x2_lo(v.x + p.x, v.y + p.y), cvt16x2_lo(v.z + p.z, v.w + p.w));
        }
      }
      *reinterpret_cast<uint2*>(a.out16p + (size_t)row * a.ld16 + j) = pp;
      if constexpr (SPLIT) *reinterpret_cast<uint2*>(a.out16p + a.lo + (size_t)row * a.ld16 + j) = ppl;
    }
    if (a.outc && a.L > 0 && l < a.Lv) {
      *reinterpret_cast<uint2*>(a.outc + crow * a.d + j) = pk;
      if constexpr (SPLIT) *reinterpret_cast<uint2*>(a.outc + a.lo + crow * a.d + j) = pkl;
    }
  }
  __device__ __forceinline__ void store1(int j, float v) const {
    if (a.out32) a.out32[(size_t)row * a.d + j] = v;
    if (a.mul32) v *= a.mul32[(size_t)row * a.d + j];
    else if (a.drop.on) v *= drop_mul1(drop_with_seed(a.drop, seed), (unsigned int)row, (unsigned int)j);
    if constexpr (SPLIT) {
      const uint16_t h = cvt16(v, a.fmt), hl = cvt16_lo(v);
      if (a.out16) {
        a.out16[(size_t)row * a.ld16 + j] = h;
        a.out16[a.lo + (size_t)row * a.ld16 + j] = hl;
      }
      if (a.out16p) {
        float vp = v;
        if (has_pos) vp = v + a.pos[prow * a.d + j];
        if (TXT && a.L > 0 && l >= a.Lv) vp = v + a.pos_txt[trow * a.d + j];
        a.out16p[(size_t)row * a.ld16 + j] = cvt16(vp, a.fmt);
        a.out16p[a.lo + (size_t)row * a.ld16 + j] = cvt16_lo(vp);
      }
      if (a.outc && a.L > 0 && l < a.Lv) {
        a.outc[crow * a.d + j] = h;
        a.outc[a.lo + crow * a.d + j] = hl;
      }
      return;
    }
    const uint16_t h = cvt16(v, a.fmt);
    if (a.out16) a.out16[(size_t)row * a.ld16 + j] = h;
    if (a.out16p) {
      uint16_t hp = has_pos ? cvt16(v + a.pos[prow * a.d + j], a.fmt) : h;
      if constexpr (TXT) {
        if (a.L > 0 && l >= a.Lv) hp = cvt16(v + a.pos_txt[trow * a.d + j], a.fmt);
      }
      a.out16p[(size_t)row * a.ld16 + j] = hp;
    }
    if (a.outc && a.L > 0 && l < a.Lv) a.outc[crow * a.d + j] = h;
  }
};

// d == NV * 128: the row lives in registers (NV float4 per lane), one global read.
template <int NV, bool TXT, bool SPLIT = false>
__global__ void __launch_bounds__(256) layernorm_rows_vec_kernel(const LnArgs a) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a.rows) return;
  const float* x = a.in + (size_t)warp * a.ld_in;
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int j = (i * 32 + lane) * 4;
    if (a.in16 != nullptr) {  // 16-bit feature shard: 64-bit load = four features
      const uint2 w = *reinterpret_cast<const uint2*>(a.in16 + (size_t)warp * a.ld_in + j);
      v[i] = make_float4(ld16((uint16_t)(w.x & 0xffff), a.in_fmt), ld16((uint16_t)(w.x >> 16), a.in_fmt),
                         ld16((uint16_t)(w.y & 0xffff), a.in_fmt), ld16((uint16_t)(w.y >> 16), a.in_fmt));
    } else
    v[i] = *reinterpret_cast<const float4*>(x + j);
    if (a.add16) {
      const uint2 h = *reinterpret_cast<const uint2*>(a.add16 + (size_t)warp * a.ld_add16 + j);
      if constexpr (SPLIT) {
        const uint2 hl = *reinterpret_cast<const uint2*>(a.add16 + a.lo + (size_t)warp * a.ld_add16 + j);
        v[i].x += ld16x3((uint16_t)(h.x & 0xffff), (uint16_t)(hl.x & 0xffff));
        v[i].y += ld16x3((uint16_t)(h.x >> 16), (uint16_t)(hl.x >> 16));
        v[i].z += ld16x3((uint16_t)(h.y & 0xffff), (uint16_t)(hl.y & 0xffff));
        v[i].w += ld16x3((uint16_t)(h.y >> 16), (uint16_t)(hl.y >> 16));
      } else {
        v[i].x += ld16((uint16_t)(h.x & 0xffff), a.fmt);
        v[i].y += ld16((uint16_t)(h.x >> 16), a.fmt);
        v[i].z += ld16((uint16_t)(h.y & 0xffff), a.fmt);
        v[i].w += ld16((uint16_t)(h.y >> 16), a.fmt);
      }
      if (a.sum_out) *reinterpret_cast<float4*>(a.sum_out + (size_t)warp * a.d + j) = v[i];
    }
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = warp_sum(s) / (float)a.d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
    q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
  }
  const float var = warp_sum(q) / (float)a.d;
  const float rstd = rsqrtf(var + a.eps);
  if (lane == 0) {
    if (a.mean_out) a.mean_out[warp] = mean;
    if (a.rstd_out) a.rstd_out[warp] = rstd;
  }
  const LnStore<TXT, SPLIT> st(a, warp);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int j = (i * 32 + lane) * 4;
    const float4 g = *reinterpret_cast<const float4*>(a.gamma + j);
    const float4 be = *reinterpret_cast<const float4*>(a.beta + j);
    float4 o;
    o.x = (v[i].x - mean) * rstd * g.x + be.x;
    o.y = (v[i].y - mean) * rstd * g.y + be.y;
    o.z = (v[i].z - mean) * rstd * g.z + be.z;
    o.w = (v[i].w - mean) * rstd * g.w + be.w;
    st.store4(j, o);
  }
}

// arbitrary d (e.g. 2818 = SlowFast+CLIP+TEF): three passes over the row, later passes hit L1/L2.
template <bool SPLIT = false>
__global__ void __launch_bounds__(256) layernorm_rows_generic_kernel(const LnArgs a) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a.rows) return;
  const float* x = a.in + (size_t)warp * a.ld_in;
  const uint16_t* x16 = a.in16 ? a.in16 + (size_t)warp * a.ld_in : nullptr;
  auto X = [&](int j) { return x16 ? ld16(x16[j], a.in_fmt) : x[j]; };
  float s = 0.f;
  for (int j = lane; j < a.d; j += 32) s += X(j);
  const float mean = warp_sum(s) / (float)a.d;
  float q = 0.f;
  for (int j = lane; j < a.d; j += 32) {
    const float dx = X(j) - mean;
    q += dx * dx;
  }
  const float var = warp_sum(q) / (float)a.d;
  const float rstd = rsqrtf(var + a.eps);
  if (lane == 0) {
    if (a.mean_out) a.mean_out[warp] = mean;
    if (a.rstd_out) a.rstd_out[warp] = rstd;
  }
  const LnStore<false, SPLIT> st(a, warp);
  for (int j = lane; j < a.d; j += 32) st.store1(j, (X(j) - mean) * rstd * a.gamma[j] + a.beta[j]);
  // zero the K padding of the 16-bit operand row (columns d .. ld16)
  if (a.out16)
    for (int j = a.d + lane; j < a.ld16; j += 32) {
      a.out16[(size_t)warp * a.ld16 + j] = 0;
      if constexpr (SPLIT) a.out16[a.lo + (size_t)warp * a.ld16 + j] = 0;
    }
}

// arbitrary d <= 128*EPT: one 128-thread block per row, the row lives in registers (single HBM read).
template <int EPT, bool TXT, bool SPLIT = false>
__global__ void __launch_bounds__(128) layernorm_rows_block_kernel(const LnArgs a) {
  pdl_prologue();
  __shared__ float s_red[4];
  __shared__ float s_stat[2];
  const int row = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* x = a.in + (size_t)row * a.ld_in;
  const uint16_t* x16 = a.in16 ? a.in16 + (size_t)row * a.ld_in : nullptr;
  float v[EPT];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < EPT; ++i) {
    const int j = tid + 128 * i;
    v[i] = j < a.d ? (x16 ? ld16(x16[j], a.in_fmt) : x[j]) : 0.f;
    if (a.add16 && j < a.d) {
      if constexpr (SPLIT)
        v[i] += ld16x3(a.add16[(size_t)row * a.ld_add16 + j], a.add16[a.lo + (size_t)row * a.ld_add16 + j]);
      else
        v[i] += ld16(a.add16[(size_t)row * a.ld_add16 + j], a.fmt);
      if (a.sum_out) a.sum_out[(size_t)row * a.d + j] = v[i];
    }
    s += v[i];
  }
  s = warp_sum(s);
  if (lane == 0) s_red[warp] = s;
  __syncthreads();
  if (tid == 0) s_stat[0] = (s_red[0] + s_red[1] + s_red[2] + s_red[3]) / (float)a.d;
  __syncthreads();
  const float mean = s_stat[0];
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < EPT; ++i) {
    const int j = tid + 128 * i;
    const float dx = j < a.d ? v[i] - mean : 0.f;
    q += dx * dx;
  }
  q = warp_sum(q);
  __syncthreads();
  if (lane == 0) s_red[warp] = q;
  __syncthreads();
  if (tid == 0) {
    const float var = (s_red[0] + s_red[1] + s_red[2] + s_red[3]) / (float)a.d;
    s_stat[1] = rsqrtf(var + a.eps);
    if (a.mean_out) a.mean_out[row] = mean;
    if (a.rstd_out) a.rstd_out[row] = s_stat[1];
  }
  __syncthreads();
  const float rstd = s_stat[1];
  const LnStore<TXT, SPLIT> st(a, row);
#pragma unroll
  for (int i = 0; i < EPT; ++i) {
    const int j = tid + 128 * i;
    if (j < a.d) st.store1(j, (v[i] - mean) * rstd * a.gamma[j] + a.beta[j]);
  }
  if (a.out16)
    for (int j = a.d + tid; j < a.ld16; j += 128) {
      a.out16[(size_t)row * a.ld16 + j] = 0;
      if constexpr (SPLIT) a.out16[a.lo + (size_t)row * a.ld16 + j] = 0;
    }
}

// even d <= 256*EPT2 with 8-byte aligned rows: same as the block kernel with 64-bit loads / 32-bit 16-bit-pair stores
// (the 2818-wide video features: 27 MB read once, 14 MB written).
template <int EPT2, bool SPLIT = false>
__global__ void __launch_bounds__(128) layernorm_rows_block2_kernel(const LnArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  __shared__ float s_red[4];
  __shared__ float s_stat[2];
  const int row = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* x = a.in + (size_t)row * a.ld_in;
  const uint16_t* x16 = a.in16 ? a.in16 + (size_t)row * a.ld_in : nullptr;
  // a thread owns 8 consecutive columns per step (four 64-bit loads): one Philox call decides all eight dropout multipliers
  constexpr int STEPS = EPT2 / 4;
  float2 v[EPT2];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < EPT2; ++i) {
    const int j = 8 * (tid + 128 * (i / 4)) + 2 * (i % 4);
    if (x16 != nullptr) {  // 16-bit feature shard: one 32-bit load = two features
      const uint32_t w = j < a.d ? *reinterpret_cast<const uint32_t*>(x16 + j) : 0u;
      v[i] = make_float2(ld16((uint16_t)(w & 0xffff), a.in_fmt), ld16((uint16_t)(w >> 16), a.in_fmt));
    } else {
      v[i] = j < a.d ? *reinterpret_cast<const float2*>(x + j) : make_float2(0.f, 0.f);
    }
    s += v[i].x + v[i].y;
  }
  s = warp_sum(s);
  if (lane == 0) s_red[warp] = s;
  __syncthreads();
  if (tid == 0) s_stat[0] = (s_red[0] + s_red[1] + s_red[2] + s_red[3]) / (float)a.d;
  __syncthreads();
  const float mean = s_stat[0];
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < EPT2; ++i) {
    const int j = 8 * (tid + 128 * (i / 4)) + 2 * (i % 4);
    if (j < a.d) {
      const float dx = v[i].x - mean, dy = v[i].y - mean;
      q += dx * dx + dy * dy;
    }
  }
  q = warp_sum(q);
  __syncthreads();
  if (lane == 0) s_red[warp] = q;
  __syncthreads();
  if (tid == 0) {
    const float var = (s_red[0] + s_red[1] + s_red[2] + s_red[3]) / (float)a.d;
    s_stat[1] = rsqrtf(var + a.eps);
    if (a.mean_out) a.mean_out[row] = mean;
    if (a.rstd_out) a.rstd_out[row] = s_stat[1];
  }
  __syncthreads();
  const float rstd = s_stat[1];
#pragma unroll
  for (int st = 0; st < STEPS; ++st) {
    const int j0 = 8 * (tid + 128 * st);
    float m8[8];
    const bool rnd = a.mul32 == nullptr && drop.on && j0 < a.d;
    if (rnd) drop_mul8(drop, (unsigned int)row, (unsigned int)(j0 >> 3), m8);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = st * 4 + k, j = j0 + 2 * k;
      if (j < a.d) {
        const float2 g = *reinterpret_cast<const float2*>(a.gamma + j);
        const float2 be = *reinterpret_cast<const float2*>(a.beta + j);
        float ox = (v[i].x - mean) * rstd * g.x + be.x;
        float oy = (v[i].y - mean) * rstd * g.y + be.y;
        if (a.mul32) {
          const float2 m = *reinterpret_cast<const float2*>(a.mul32 + (size_t)row * a.d + j);
          ox *= m.x;
          oy *= m.y;
        } else if (rnd) {
          ox *= m8[2 * k];
          oy *= m8[2 * k + 1];
        }
        *reinterpret_cast<uint32_t*>(a.out16 + (size_t)row * a.ld16 + j) = cvt16x2(ox, oy, a.fmt);
        if constexpr (SPLIT) *reinterpret_cast<uint32_t*>(a.out16 + a.lo + (size_t)row * a.ld16 + j) = cvt16x2_lo(ox, oy);
      }
    }
  }
  for (int j = a.d + 2 * tid; j < a.ld16; j += 256) {
    *reinterpret_cast<uint32_t*>(a.out16 + (size_t)row * a.ld16 + j) = 0u;
    if constexpr (SPLIT) *reinterpret_cast<uint32_t*>(a.out16 + a.lo + (size_t)row * a.ld16 + j) = 0u;
  }
}

template <bool SPLIT>
static int launch_layernorm_impl(const LnArgs& a, cudaStream_t stream, int* kernel_used) {
  const int threads = 256;
  const int blocks = (a.rows * 32 + threads - 1) / threads;
  const bool vec_ok = (a.ld_in % 4 == 0) && (a.ld16 == a.d) &&
                      (a.in16 ? (reinterpret_cast<uintptr_t>(a.in16) & 7) == 0 : (reinterpret_cast<uintptr_t>(a.in) & 15) == 0);
  int k;
  if (a.pos_txt != nullptr) {  // LayerNorm 2 of an encoder layer with learned text positions (out16p of the next layer)
    if (!a.out16p || a.L <= 0 || a.d > 128 * 24) {
      set_error("layernorm: text positions need the structured q/k operand and d <= 3072");
      return (int)cudaErrorInvalidValue;
    }
    if (vec_ok && a.d == 1024) k = LN_VEC8_TXT;
    else if (vec_ok && a.d == 512) k = LN_VEC4_TXT;
    else if (vec_ok && a.d == 256) k = LN_VEC2_TXT;
    else if (a.d <= 128 * 8) k = LN_BLOCK8_TXT;
    else k = LN_BLOCK24_TXT;
  } else if (vec_ok && a.d == 1024) k = LN_VEC8;
  else if (vec_ok && a.d == 512) k = LN_VEC4;
  else if (vec_ok && a.d == 256) k = LN_VEC2;
  else if (a.d > 1024 && a.d <= 1024 * 3 && a.d % 2 == 0 && a.ld_in % 2 == 0 && a.ld16 % 2 == 0 && a.out16 && !a.out32 &&
           !a.out16p && !a.outc && !a.add16 && (a.in16 ? (reinterpret_cast<uintptr_t>(a.in16) & 3) == 0 : (reinterpret_cast<uintptr_t>(a.in) & 7) == 0) &&
           (reinterpret_cast<uintptr_t>(a.gamma) & 7) == 0 && (reinterpret_cast<uintptr_t>(a.beta) & 7) == 0 &&
           (!a.mul32 || (reinterpret_cast<uintptr_t>(a.mul32) & 7) == 0))
    k = LN_BLOCK2_12;
  else if (a.d <= 128 * 8) k = LN_BLOCK8;
  else if (a.d <= 128 * 24) k = LN_BLOCK24;
  else {
    if (a.add16) {
      set_error("layernorm: fused branch add needs d <= 3072");
      return (int)cudaErrorInvalidValue;
    }
    k = LN_GENERIC;
  }
  const dim3 vec_grid(blocks), vec_block(threads), row_grid(a.rows), row_block(128);
  switch (k) {
    case LN_VEC8: launch_k(layernorm_rows_vec_kernel<8, false, SPLIT>, vec_grid, vec_block, 0, stream, a); break;
    case LN_VEC4: launch_k(layernorm_rows_vec_kernel<4, false, SPLIT>, vec_grid, vec_block, 0, stream, a); break;
    case LN_VEC2: launch_k(layernorm_rows_vec_kernel<2, false, SPLIT>, vec_grid, vec_block, 0, stream, a); break;
    case LN_VEC8_TXT: launch_k(layernorm_rows_vec_kernel<8, true, SPLIT>, vec_grid, vec_block, 0, stream, a); break;
    case LN_VEC4_TXT: launch_k(layernorm_rows_vec_kernel<4, true, SPLIT>, vec_grid, vec_block, 0, stream, a); break;
    case LN_VEC2_TXT: launch_k(layernorm_rows_vec_kernel<2, true, SPLIT>, vec_grid, vec_block, 0, stream, a); break;
    case LN_BLOCK8: launch_k(layernorm_rows_block_kernel<8, false, SPLIT>, row_grid, row_block, 0, stream, a); break;
    case LN_BLOCK24: launch_k(layernorm_rows_block_kernel<24, false, SPLIT>, row_grid, row_block, 0, stream, a); break;
    case LN_BLOCK8_TXT: launch_k(layernorm_rows_block_kernel<8, true, SPLIT>, row_grid, row_block, 0, stream, a); break;
    case LN_BLOCK24_TXT: launch_k(layernorm_rows_block_kernel<24, true, SPLIT>, row_grid, row_block, 0, stream, a); break;
    case LN_BLOCK2_12: launch_k(layernorm_rows_block2_kernel<12, SPLIT>, row_grid, row_block, 0, stream, a); break;
    default: launch_k(layernorm_rows_generic_kernel<SPLIT>, vec_grid, vec_block, 0, stream, a); break;
  }
  if (kernel_used) *kernel_used = k + (SPLIT ? LN_SPLIT : 0);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("layernorm launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

int launch_layernorm(const LnArgs& a, cudaStream_t stream, int* kernel_used) {
  if (a.rows <= 0) return 0;
  if (a.split) {
    if (a.fmt != 0 || a.mul32 != nullptr || a.drop.on) {
      set_error("layernorm: fp16x3 output needs fmt 0 and no dropout");
      return (int)cudaErrorInvalidValue;
    }
    return launch_layernorm_impl<true>(a, stream, kernel_used);
  }
  return launch_layernorm_impl<false>(a, stream, kernel_used);
}

// ------------------------------------------------------------------------------------------------
// Learned text positions (TxtPosArgs, rowops.h).  One warp per text row; lane owns columns 2 (lane + 32 i), i < d / 64.
// ------------------------------------------------------------------------------------------------
constexpr int kTxtPosMaxPairs = 16;  // d <= 64 * 16
template <bool SPLIT = false>
__global__ void __launch_bounds__(256) txt_pos_rows_kernel(const TxtPosArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= a.B * a.Lt) return;
  const int b = row / a.Lt, l = row - b * a.Lt;
  const int npairs = a.d >> 6;
  const float* x = a.xt + (size_t)row * a.d;
  const float* P = a.table + (size_t)l * a.d;
  float2 u[kTxtPosMaxPairs];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kTxtPosMaxPairs; ++i) {
    if (i < npairs) {
      const int j = 2 * (lane + 32 * i);
      const float2 xv = *reinterpret_cast<const float2*>(x + j);
      const float2 pv = *reinterpret_cast<const float2*>(P + j);
      u[i] = make_float2(xv.x + pv.x, xv.y + pv.y);
      s += u[i].x + u[i].y;
    }
  }
  const float mean = warp_sum(s) / (float)a.d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kTxtPosMaxPairs; ++i) {
    if (i < npairs) {
      const float dx = u[i].x - mean, dy = u[i].y - mean;
      q += dx * dx + dy * dy;
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)a.d + 1e-5f);
  if (lane == 0 && a.mean_out) {
    a.mean_out[row] = mean;
    a.rstd_out[row] = rstd;
  }
  uint16_t* xp = a.xpos16 + ((size_t)b * a.L + a.Lv + l) * a.d;
#pragma unroll
  for (int i = 0; i < kTxtPosMaxPairs; ++i) {
    if (i < npairs) {
      const int j = 2 * (lane + 32 * i);
      const float2 g = *reinterpret_cast<const float2*>(a.gamma + j);
      const float2 be = *reinterpret_cast<const float2*>(a.beta + j);
      float ox = (u[i].x - mean) * rstd * g.x + be.x;
      float oy = (u[i].y - mean) * rstd * g.y + be.y;
      if (a.mul32) {
        const float2 m = *reinterpret_cast<const float2*>(a.mul32 + (size_t)row * a.d + j);
        ox *= m.x;
        oy *= m.y;
      } else if (drop.on) {
        ox *= drop_mul1(drop, (unsigned int)row, (unsigned int)j);
        oy *= drop_mul1(drop, (unsigned int)row, (unsigned int)(j + 1));
      }
      *reinterpret_cast<float2*>(a.pos + (size_t)row * a.d + j) = make_float2(ox, oy);
      const float2 xv = *reinterpret_cast<const float2*>(x + j);
      *reinterpret_cast<uint32_t*>(xp + j) = cvt16x2(xv.x + ox, xv.y + oy, a.fmt);
      if constexpr (SPLIT) *reinterpret_cast<uint32_t*>(xp + a.lo + j) = cvt16x2_lo(xv.x + ox, xv.y + oy);
    }
  }
}

int launch_txt_pos(const TxtPosArgs& a, cudaStream_t stream) {
  if (a.d % 64 != 0 || a.d > 64 * kTxtPosMaxPairs) {
    set_error("text positions: hidden_dim %d must be a multiple of 64 and <= %d", a.d, 64 * kTxtPosMaxPairs);
    return (int)cudaErrorInvalidValue;
  }
  const int rows = a.B * a.Lt;
  if (a.split) launch_k(txt_pos_rows_kernel<true>, dim3((rows * 32 + 255) / 256), dim3(256), 0, stream, a);
  else launch_k(txt_pos_rows_kernel<false>, dim3((rows * 32 + 255) / 256), dim3(256), 0, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("txt_pos launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// Sine position table  pos[b, l, j]  (fp32, [B*Lv, d])
//   c = cumsum(mask); e = c / (c_last + 1e-6) * 2pi; pos = sin(e / dim_t[j]) (j even) | cos(e / dim_t[j]) (j odd)
// dim_t is supplied by the host (computed once with the reference's own fp32 expression).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sine_pos_table_kernel(const float* __restrict__ mask, const float* __restrict__ txt_mask,
                                                            const float* __restrict__ dim_t, float* __restrict__ pos,
                                                            float* __restrict__ key_mask, int Lv, int Lt, int d,
                                                            float* __restrict__ dp_out, int dp_n, unsigned long long dp_seed,
                                                            const unsigned long long* __restrict__ dp_seed_ptr, float dp_keep) {
  pdl_prologue();
  if (dp_out != nullptr && blockIdx.x == 0 && blockIdx.y == 0) {  // DropPath scales of this step ([sites, B], a few hundred values)
    const unsigned long long seed = dp_seed_of(dp_seed, dp_seed_ptr);
    for (int i = threadIdx.x; i < dp_n; i += 256) dp_out[i] = droppath_scale(seed, (unsigned int)i, dp_keep);
  }
  extern __shared__ float s_e[];  // [Lv] cumulative position, then the normalised angle
  __shared__ float s_part[256];
  const int b = blockIdx.x;
  const int tid = threadIdx.x;
  // block-wide inclusive scan of the 0/1 mask (sums of small integers: exact in fp32 in any order)
  const int per = (Lv + 255) / 256;
  const int l0 = tid * per;
  float run = 0.f;
  for (int l = l0; l < min(Lv, l0 + per); ++l) {
    run += mask[(size_t)b * Lv + l];
    s_e[l] = run;
  }
  s_part[tid] = run;
  __syncthreads();
  if (tid == 0) {
    float acc = 0.f;
    for (int i = 0; i < 256; ++i) {
      const float t = s_part[i];
      s_part[i] = acc;
      acc += t;
    }
  }
  __syncthreads();
  const float off = s_part[tid];
  for (int l = l0; l < min(Lv, l0 + per); ++l) s_e[l] += off;
  __syncthreads();
  const float denom = s_e[Lv - 1] + 1e-6f;
  const float scale = 6.283185307179586f;  // float32(2*math.pi)
  __syncthreads();
  for (int l = tid; l < Lv; l += 256) s_e[l] = s_e[l] / denom * scale;
  // concatenated key mask [B, Lv+Lt] (mask = cat([src_vid_mask, src_txt_mask]), model/univtg.py:120)
  if (key_mask != nullptr && blockIdx.y == 0) {
    const int L = Lv + Lt;
    for (int l = tid; l < L; l += 256)
      key_mask[(size_t)b * L + l] = (l < Lv) ? mask[(size_t)b * Lv + l] : txt_mask[(size_t)b * Lt + (l - Lv)];
  }
  __syncthreads();
  // dim_t[2k] == dim_t[2k+1]: one division and one sincos give the (sin, cos) pair of columns 2k, 2k+1
  const int half = d >> 1;
  const int total = Lv * half;
  for (int i = blockIdx.y * 256 + tid; i < total; i += gridDim.y * 256) {
    const int l = i / half;
    const int k = i - l * half;
    const float arg = s_e[l] / dim_t[2 * k];
    float sv, cv;
    sincosf(arg, &sv, &cv);
    *reinterpret_cast<float2*>(pos + ((size_t)b * Lv + l) * d + 2 * k) = make_float2(sv, cv);
  }
}

int launch_sine_pos(const float* mask, const float* txt_mask, const float* dim_t, float* pos, float* key_mask, int B, int Lv,
                    int Lt, int d, cudaStream_t stream, float* dp_out, int dp_sites, unsigned long long dp_seed, float dp_keep,
                    const unsigned long long* dp_seed_ptr) {
  int chunks = (Lv * d + 4095) / 4096;
  if (chunks < 1) chunks = 1;
  if (chunks > 128) chunks = 128;
  launch_k(sine_pos_table_kernel, dim3(dim3(B, chunks)), dim3(256), Lv * sizeof(float), stream, mask, txt_mask, dim_t, pos, key_mask, Lv, Lt, d,
           dp_out, dp_sites * B, dp_seed, dp_seed_ptr, dp_keep);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("sine_pos launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

__global__ void __launch_bounds__(256) dropout_mask_kernel(const DropSpec spec_in, size_t n, size_t cols, float* __restrict__ out) {
  pdl_prologue();
  const DropSpec spec = drop_resolve(spec_in);
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256)
    out[i] = spec.on ? drop_mul1(spec, (unsigned int)(i / cols), (unsigned int)(i % cols)) : 1.f;
}
__global__ void __launch_bounds__(256) droppath_scales_kernel(unsigned long long seed_in, const unsigned long long* __restrict__ seed_ptr,
                                                             int n, float keep, float* __restrict__ out) {
  pdl_prologue();
  const unsigned long long seed = dp_seed_of(seed_in, seed_ptr);
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) out[i] = droppath_scale(seed, (unsigned int)i, keep);
}
__global__ void __launch_bounds__(32) rng_advance_kernel(unsigned long long base, unsigned long long* __restrict__ counter,
                                                         unsigned long long* __restrict__ seed) {
  pdl_prologue();
  if (threadIdx.x == 0) {
    const unsigned long long k = *counter + 1ull;
    *counter = k;
    *seed = rng_seed_at(base, k);
  }
}
int launch_rng_advance(unsigned long long base, unsigned long long* counter, unsigned long long* seed, cudaStream_t stream) {
  launch_k(rng_advance_kernel, dim3(1), dim3(32), 0, stream, base, counter, seed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("rng_advance launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}
int launch_dropout_mask(const DropSpec& spec, size_t n, size_t cols, float* out, cudaStream_t stream) {
  if (n == 0) return 0;
  size_t blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_k(dropout_mask_kernel, dim3((unsigned)blocks), dim3(256), 0, stream, spec, n, cols, out);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("dropout_mask launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}
int launch_droppath_scales(unsigned long long seed, int n, float keep, float* out, cudaStream_t stream, const unsigned long long* seed_ptr) {
  if (n <= 0) return 0;
  launch_k(droppath_scales_kernel, dim3((n + 255) / 256), dim3(256), 0, stream, seed, seed_ptr, n, keep, out);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("droppath_scales launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// WeightedPool + cosine saliency.  One CTA per sample.
//   alpha = softmax_l(x_t . w + (1 - m_t) * -1e30);  pooled = sum_l alpha_l x_t[l]
//   sal[l] = cos(x_v[l], pooled) + log(m_v[l] + 1e-45)      (denormal-sensitive: no FTZ / fast-math)
// ------------------------------------------------------------------------------------------------
// logits[b, l] = x_t[b, l] . w + (1 - mask) * -1e30: one warp per text token
__global__ void __launch_bounds__(256) pool_logits_kernel(const PoolSalArgs a, float* __restrict__ logits) {
  pdl_prologue();
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= a.B * a.Lt) return;
  const float* x = a.x_txt + (size_t)gw * a.d;
  float s = 0.f;
  for (int j = lane * 4; j < a.d; j += 128) {
    const float4 v = *reinterpret_cast<const float4*>(x + j);
    const float4 w = *reinterpret_cast<const float4*>(a.w + j);
    s += v.x * w.x + v.y * w.y + v.z * w.z + v.w * w.w;
  }
  s = warp_sum(s);
  if (lane == 0) logits[gw] = s + (1.0f - a.txt_mask[gw]) * (-1e30f);
}

// softmax over the tokens (recomputed per block, Lt is small) and pooled[b, j] for a 128-column slab
__global__ void __launch_bounds__(128) weighted_pool_kernel(const PoolSalArgs a, const float* __restrict__ logits) {
  pdl_prologue();
  extern __shared__ float s_alpha[];  // [Lt]
  __shared__ float s_stat[2];
  const int b = blockIdx.x;
  const int j = blockIdx.y * 128 + threadIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0) {
    float mx = -INFINITY;
    for (int l = lane; l < a.Lt; l += 32) mx = fmaxf(mx, logits[(size_t)b * a.Lt + l]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int l = lane; l < a.Lt; l += 32) {
      const float e = expf(logits[(size_t)b * a.Lt + l] - mx);
      s_alpha[l] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    if (lane == 0) s_stat[0] = sum;
  }
  __syncthreads();
  const float inv = s_stat[0];
  for (int l = threadIdx.x; l < a.Lt; l += 128) {  // each element is read and written by the same thread
    const float al = s_alpha[l] / inv;
    s_alpha[l] = al;
    if (a.alpha_out && blockIdx.y == 0) a.alpha_out[(size_t)b * a.Lt + l] = al;
  }
  __syncthreads();
  if (j < a.d) {
    const float* xt = a.x_txt + (size_t)b * a.Lt * a.d + j;
    float p = 0.f;
    for (int l = 0; l < a.Lt; ++l) p += xt[(size_t)l * a.d] * s_alpha[l];
    a.pooled[(size_t)b * a.d + j] = p;
  }
}

// one warp per (b, l): cos(x_v[b,l], pooled[b]) + log(mask + 1e-45)
__global__ void __launch_bounds__(256) cosine_saliency_kernel(const PoolSalArgs a) {
  pdl_prologue();
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= a.B * a.Lv) return;
  const int b = gw / a.Lv;
  const float* xv = a.x_vid + (size_t)gw * a.d;
  const float* pl = a.pooled + (size_t)b * a.d;
  float dot = 0.f, nn = 0.f, pn = 0.f;
  for (int j = lane * 4; j < a.d; j += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xv + j);
    const float4 p = *reinterpret_cast<const float4*>(pl + j);
    dot += v.x * p.x + v.y * p.y + v.z * p.z + v.w * p.w;
    nn += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    pn += p.x * p.x + p.y * p.y + p.z * p.z + p.w * p.w;
  }
  dot = warp_sum(dot);
  nn = warp_sum(nn);
  pn = warp_sum(pn);
  if (lane == 0) {
    const float vn = fmaxf(sqrtf(nn), 1e-8f);
    const float pnorm = fmaxf(sqrtf(pn), 1e-8f);
    a.saliency[gw] = dot / (vn * pnorm) + logf(a.vid_mask[gw] + 1e-45f);
  }
}

int launch_pool_saliency(const PoolSalArgs& a, cudaStream_t stream) {
  launch_k(pool_logits_kernel, dim3((a.B * a.Lt * 32 + 255) / 256), dim3(256), 0, stream, a, a.logits_ws);
  launch_k(weighted_pool_kernel, dim3(dim3(a.B, (a.d + 127) / 128)), dim3(128), (size_t)a.Lt * sizeof(float), stream, a, a.logits_ws);
  const int rows = a.B * a.Lv;
  launch_k(cosine_saliency_kernel, dim3((rows * 32 + 255) / 256), dim3(256), 0, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("pool_saliency launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// Final conv layer of both heads (out channels 1 and 2) + sigmoid + sign.  One warp per (b, l).
// Hidden activations are 16-bit in the separated conv layout: row 1 + b*(Lv+1) + l, zero separator rows.
// ------------------------------------------------------------------------------------------------
// SPLIT: the hidden activations are fp16x3 pairs (lo plane a.lo elements after the hi plane).
template <bool SPLIT = false>
__global__ void __launch_bounds__(256) conv_head_final_kernel(const HeadFinalArgs a) {
  pdl_prologue();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a.B * a.Lv) return;
  const int b = warp / a.Lv, l = warp - b * a.Lv;
  const size_t row = (size_t)1 + (size_t)b * (a.Lv + 1) + l;  // centre row in the +1-offset buffer
  float acc_c = 0.f, acc_s0 = 0.f, acc_s1 = 0.f;
  for (int t = 0; t < 3; ++t) {
    const uint16_t* hc = a.h_cls + (row + t - 1) * a.d;
    const uint16_t* hs = a.h_span + (row + t - 1) * a.d;
    const float* wc = a.w_cls + (size_t)t * a.d;            // [3][d]
    const float* ws0 = a.w_span + (size_t)t * a.d;          // [2][3][d]
    const float* ws1 = a.w_span + (size_t)(3 + t) * a.d;
    for (int j = lane * 2; j < a.d; j += 64) {
      const uint32_t c2 = *reinterpret_cast<const uint32_t*>(hc + j);
      const uint32_t s2 = *reinterpret_cast<const uint32_t*>(hs + j);
      float c0 = ld16((uint16_t)(c2 & 0xffff), a.fmt), c1 = ld16((uint16_t)(c2 >> 16), a.fmt);
      float s0 = ld16((uint16_t)(s2 & 0xffff), a.fmt), s1 = ld16((uint16_t)(s2 >> 16), a.fmt);
      if constexpr (SPLIT) {
        const uint32_t c2l = *reinterpret_cast<const uint32_t*>(hc + a.lo + j);
        const uint32_t s2l = *reinterpret_cast<const uint32_t*>(hs + a.lo + j);
        c0 = ld16x3((uint16_t)(c2 & 0xffff), (uint16_t)(c2l & 0xffff));
        c1 = ld16x3((uint16_t)(c2 >> 16), (uint16_t)(c2l >> 16));
        s0 = ld16x3((uint16_t)(s2 & 0xffff), (uint16_t)(s2l & 0xffff));
        s1 = ld16x3((uint16_t)(s2 >> 16), (uint16_t)(s2l >> 16));
      }
      acc_c += c0 * wc[j] + c1 * wc[j + 1];
      acc_s0 += s0 * ws0[j] + s1 * ws0[j + 1];
      acc_s1 += s0 * ws1[j] + s1 * ws1[j + 1];
    }
  }
  acc_c = warp_sum(acc_c);
  acc_s0 = warp_sum(acc_s0);
  acc_s1 = warp_sum(acc_s1);
  if (lane == 0) {
    const float zc = acc_c + a.b_cls[0];
    const float z0 = acc_s0 + a.b_span[0];
    const float z1 = acc_s1 + a.b_span[1];
    a.pred_logits[warp] = 1.f / (1.f + expf(-zc));
    a.pred_spans[(size_t)warp * 2 + 0] = -(1.f / (1.f + expf(-z0)));
    a.pred_spans[(size_t)warp * 2 + 1] = 1.f / (1.f + expf(-z1));
  }
}

int launch_conv_head_final(const HeadFinalArgs& a, cudaStream_t stream) {
  const int rows = a.B * a.Lv;
  const int threads = 256;
  const int blocks = (rows * 32 + threads - 1) / threads;
  if (a.split) launch_k(conv_head_final_kernel<true>, dim3(blocks), dim3(threads), 0, stream, a);
  else launch_k(conv_head_final_kernel<false>, dim3(blocks), dim3(threads), 0, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("conv_head_final launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

}  // namespace uv
