// Bandwidth-bound backward kernels of the UniVTG hot path (SURVEY.md A.6): LayerNorm backward, 16-bit conversion with
// bias-gradient column sums, the last conv layer of the heads, weighted-pool backward and stream-gradient assembly.
// Gradients that feed tensor-core GEMMs are emitted as bf16 (fp16 would underflow), statistics stay fp32.
#include <math.h>
#include <stdlib.h>

#include "backward.h"
#include "kernels.h"
#include "ptx.cuh"

namespace uv {

// ------------------------------------------------------------------------------------------------
// LayerNorm backward.  128 threads walk one row at a time (columns j = tid + 128 i, row in registers);
// each block owns a strided set of rows and keeps dgamma / dbeta / colsum partials in registers.
// ------------------------------------------------------------------------------------------------
template <int EPT>
__global__ void __launch_bounds__(128) layernorm_bwd_kernel(const LnBwdArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  __shared__ float s_red[2][4];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float acc_g[EPT], acc_b[EPT], acc_c[EPT];
#pragma unroll
  for (int i = 0; i < EPT; ++i) acc_g[i] = acc_b[i] = acc_c[i] = 0.f;
  const float inv_d = 1.0f / (float)a.d;

  for (int row = blockIdx.x; row < a.rows; row += gridDim.x) {
    const float mean = a.mean[row], rstd = a.rstd[row];
    const float* dout = a.dout + (size_t)row * a.ld_dout;
    const float* y = a.y + (size_t)row * a.ld_y;
    float xh[EPT], g[EPT];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const int j = tid + 128 * i;
      xh[i] = 0.f;
      g[i] = 0.f;
      if (j < a.d) {
        float dj = dout[j];
        if (a.dout_mul) dj *= a.dout_mul[(size_t)row * a.d + j];
        else if (drop.on) dj *= drop_mul1(drop, (unsigned int)row, (unsigned int)j);
        xh[i] = (y[j] - mean) * rstd;
        g[i] = dj * a.gamma[j];
        acc_g[i] += dj * xh[i];
        acc_b[i] += dj;
        s1 += g[i];
        s2 += g[i] * xh[i];
      }
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    __syncthreads();  // previous iteration's readers are done
    if (lane == 0) {
      s_red[0][warp] = s1;
      s_red[1][warp] = s2;
    }
    __syncthreads();
    const float c1 = (s_red[0][0] + s_red[0][1] + s_red[0][2] + s_red[0][3]) * inv_d;
    const float c2 = (s_red[1][0] + s_red[1][1] + s_red[1][2] + s_red[1][3]) * inv_d;
    float rs = 1.f;
    if (a.row_scale != nullptr) rs = a.row_scale[a.L > 0 ? row / a.L : 0];
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const int j = tid + 128 * i;
      if (j < a.d) {
        float dy = rstd * (g[i] - c1 - xh[i] * c2);
        if (a.relu_mask_y && !(y[j] > 0.f)) dy = 0.f;
        if (a.dy32) a.dy32[(size_t)row * a.d + j] = dy;
        const float br = dy * rs;
        acc_c[i] += br;
        if (a.dbr16) a.dbr16[(size_t)row * a.ld16 + j] = cvt16(br, a.fmt16);
      }
    }
    if (a.dbr16)
      for (int j = a.d + tid; j < a.ld16; j += 128) a.dbr16[(size_t)row * a.ld16 + j] = 0;
  }
#pragma unroll
  for (int i = 0; i < EPT; ++i) {
    const int j = tid + 128 * i;
    if (j < a.d) {
      if (a.dgamma) atomicAdd(a.dgamma + j, acc_g[i] * a.pgrad_scale);
      if (a.dbeta) atomicAdd(a.dbeta + j, acc_b[i] * a.pgrad_scale);
      if (a.colsum) atomicAdd(a.colsum + j, acc_c[i] * a.pgrad_scale);
    }
  }
}

// 128-bit variant for row lengths that are multiples of 4 (d <= 512 * NV): the next row's operands are fetched before the
// current row's block reduction so the DRAM latency of consecutive rows overlaps.
template <int NV>
__global__ void __launch_bounds__(128) layernorm_bwd_vec_kernel(const LnBwdArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  __shared__ float s_red[2][4];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float4 acc_g[NV], acc_b[NV], acc_c[NV], gam[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    acc_g[i] = acc_b[i] = acc_c[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int j = (tid + 128 * i) * 4;
    gam[i] = j < a.d ? *reinterpret_cast<const float4*>(a.gamma + j) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float inv_d = 1.0f / (float)a.d;
  float4 nd[NV], ny[NV];
  auto fetch = [&](int row) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = (tid + 128 * i) * 4;
      nd[i] = ny[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < a.rows && j < a.d) {
        nd[i] = __ldg(reinterpret_cast<const float4*>(a.dout + (size_t)row * a.ld_dout + j));
        ny[i] = __ldg(reinterpret_cast<const float4*>(a.y + (size_t)row * a.ld_y + j));
        if (a.dout_mul) {
          const float4 m = __ldg(reinterpret_cast<const float4*>(a.dout_mul + (size_t)row * a.d + j));
          nd[i].x *= m.x, nd[i].y *= m.y, nd[i].z *= m.z, nd[i].w *= m.w;
        } else if (drop.on) {
          const float4 m = drop_mul4(drop, (unsigned int)row, (unsigned int)j);
          nd[i].x *= m.x, nd[i].y *= m.y, nd[i].z *= m.z, nd[i].w *= m.w;
        }
      }
    }
  };
  fetch(blockIdx.x);
  for (int row = blockIdx.x; row < a.rows; row += gridDim.x) {
    const float mean = a.mean[row], rstd = a.rstd[row];
    float4 dj[NV], yv[NV], xh[NV], g[NV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      dj[i] = nd[i];
      yv[i] = ny[i];
    }
    fetch(row + gridDim.x);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = (tid + 128 * i) * 4;
      const bool in = j < a.d;
#define UV_LNB(c)                                          \
  xh[i].c = in ? (yv[i].c - mean) * rstd : 0.f;            \
  g[i].c = dj[i].c * gam[i].c;                             \
  acc_g[i].c += dj[i].c * xh[i].c;                         \
  acc_b[i].c += dj[i].c;                                   \
  s1 += g[i].c;                                            \
  s2 += g[i].c * xh[i].c;
      UV_LNB(x) UV_LNB(y) UV_LNB(z) UV_LNB(w)
#undef UV_LNB
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    __syncthreads();
    if (lane == 0) {
      s_red[0][warp] = s1;
      s_red[1][warp] = s2;
    }
    __syncthreads();
    const float c1 = (s_red[0][0] + s_red[0][1] + s_red[0][2] + s_red[0][3]) * inv_d;
    const float c2 = (s_red[1][0] + s_red[1][1] + s_red[1][2] + s_red[1][3]) * inv_d;
    float rs = 1.f;
    if (a.row_scale != nullptr) rs = a.row_scale[a.L > 0 ? row / a.L : 0];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = (tid + 128 * i) * 4;
      if (j < a.d) {
        float4 dy;
        dy.x = rstd * (g[i].x - c1 - xh[i].x * c2);
        dy.y = rstd * (g[i].y - c1 - xh[i].y * c2);
        dy.z = rstd * (g[i].z - c1 - xh[i].z * c2);
        dy.w = rstd * (g[i].w - c1 - xh[i].w * c2);
        if (a.relu_mask_y) {
          if (!(yv[i].x > 0.f)) dy.x = 0.f;
          if (!(yv[i].y > 0.f)) dy.y = 0.f;
          if (!(yv[i].z > 0.f)) dy.z = 0.f;
          if (!(yv[i].w > 0.f)) dy.w = 0.f;
        }
        if (a.dy32) *reinterpret_cast<float4*>(a.dy32 + (size_t)row * a.d + j) = dy;
        const float4 br = make_float4(dy.x * rs, dy.y * rs, dy.z * rs, dy.w * rs);
        acc_c[i].x += br.x, acc_c[i].y += br.y, acc_c[i].z += br.z, acc_c[i].w += br.w;
        if (a.dbr16)
          *reinterpret_cast<uint2*>(a.dbr16 + (size_t)row * a.ld16 + j) =
              make_uint2(cvt16x2(br.x, br.y, a.fmt16), cvt16x2(br.z, br.w, a.fmt16));
      }
    }
    if (a.dbr16)
      for (int j = a.d + tid; j < a.ld16; j += 128) a.dbr16[(size_t)row * a.ld16 + j] = 0;
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int j = (tid + 128 * i) * 4;
    if (j < a.d) {
      const float ps = a.pgrad_scale;
      if (a.dgamma) red_add_f32x4(a.dgamma + j, make_float4(acc_g[i].x * ps, acc_g[i].y * ps, acc_g[i].z * ps, acc_g[i].w * ps));
      if (a.dbeta) red_add_f32x4(a.dbeta + j, make_float4(acc_b[i].x * ps, acc_b[i].y * ps, acc_b[i].z * ps, acc_b[i].w * ps));
      if (a.colsum) red_add_f32x4(a.colsum + j, make_float4(acc_c[i].x * ps, acc_c[i].y * ps, acc_c[i].z * ps, acc_c[i].w * ps));
    }
  }
}

// Warp-per-row variant for d == NV * 128 (256 / 512 / 1024: every LayerNorm of the encoder and the inner projector layers).  A warp
// holds its whole row in registers, so the two row statistics are warp shuffles - no block barrier per row (the block-per-row
// kernel above spends two __syncthreads per 1024-element row).  Column partials (dgamma,
// dbeta, bias column sums) stay in registers over the rows a warp visits, are combined across the block's 8 warps through
// shared memory and leave as ONE vector reduction per block and column group.
template <int NV>
__global__ void __launch_bounds__(256) layernorm_bwd_warp_kernel(const LnBwdArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  extern __shared__ float s_part[];  // [8 warps][NV * 128] floats, reused for the three column accumulators
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int D = NV * 128;
  float4 acc_g[NV], acc_b[NV], acc_c[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) acc_g[i] = acc_b[i] = acc_c[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  const float inv_d = 1.0f / (float)D;
  for (int row = blockIdx.x * 8 + warp; row < a.rows; row += gridDim.x * 8) {
    float4 g[NV], xh[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = (i * 32 + lane) * 4;
      g[i] = __ldg(reinterpret_cast<const float4*>(a.dout + (size_t)row * a.ld_dout + j));
      xh[i] = __ldg(reinterpret_cast<const float4*>(a.y + (size_t)row * a.ld_y + j));
    }
    const float mean = a.mean[row], rstd = a.rstd[row];
    float rs = 1.f;
    if (a.row_scale != nullptr) rs = a.row_scale[a.L > 0 ? row / a.L : 0];
    float s1 = 0.f, s2 = 0.f;
    unsigned int relu = 0u;  // bit 4 i + c: y > 0 (ReLU mask of the projector chain)
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = (i * 32 + lane) * 4;
      if (a.dout_mul) {
        const float4 m = __ldg(reinterpret_cast<const float4*>(a.dout_mul + (size_t)row * D + j));
        g[i].x *= m.x, g[i].y *= m.y, g[i].z *= m.z, g[i].w *= m.w;
      } else if (drop.on) {
        const float4 m = drop_mul4(drop, (unsigned int)row, (unsigned int)j);
        g[i].x *= m.x, g[i].y *= m.y, g[i].z *= m.z, g[i].w *= m.w;
      }
      const float4 gam = __ldg(reinterpret_cast<const float4*>(a.gamma + j));
#define UV_LNW(c, bit)                                  \
  if (xh[i].c > 0.f) relu |= 1u << (4 * i + bit);       \
  xh[i].c = (xh[i].c - mean) * rstd;                    \
  acc_g[i].c += g[i].c * xh[i].c;                       \
  acc_b[i].c += g[i].c;                                 \
  g[i].c *= gam.c;                                      \
  s1 += g[i].c;                                         \
  s2 += g[i].c * xh[i].c;
      UV_LNW(x, 0) UV_LNW(y, 1) UV_LNW(z, 2) UV_LNW(w, 3)
#undef UV_LNW
    }
    const float c1 = warp_sum(s1) * inv_d, c2 = warp_sum(s2) * inv_d;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int j = (i * 32 + lane) * 4;
      float4 dy;
      dy.x = rstd * (g[i].x - c1 - xh[i].x * c2);
      dy.y = rstd * (g[i].y - c1 - xh[i].y * c2);
      dy.z = rstd * (g[i].z - c1 - xh[i].z * c2);
      dy.w = rstd * (g[i].w - c1 - xh[i].w * c2);
      if (a.relu_mask_y) {
        if (!(relu & (1u << (4 * i + 0)))) dy.x = 0.f;
        if (!(relu & (1u << (4 * i + 1)))) dy.y = 0.f;
        if (!(relu & (1u << (4 * i + 2)))) dy.z = 0.f;
        if (!(relu & (1u << (4 * i + 3)))) dy.w = 0.f;
      }
      if (a.dy32) *reinterpret_cast<float4*>(a.dy32 + (size_t)row * D + j) = dy;
      const float4 br = make_float4(dy.x * rs, dy.y * rs, dy.z * rs, dy.w * rs);
      acc_c[i].x += br.x, acc_c[i].y += br.y, acc_c[i].z += br.z, acc_c[i].w += br.w;
      if (a.dbr16)
        *reinterpret_cast<uint2*>(a.dbr16 + (size_t)row * a.ld16 + j) = make_uint2(cvt16x2(br.x, br.y, a.fmt16), cvt16x2(br.z, br.w, a.fmt16));
    }
  }
  // block-level combination of the column partials: warp w parks its slice, 256 threads sum the 8 slices of 4 columns each
  auto flush = [&](const float4 (&acc)[NV], float* dst) {
    if (dst == nullptr) return;  // uniform over the block
    __syncthreads();
#pragma unroll
    for (int i = 0; i < NV; ++i) *reinterpret_cast<float4*>(s_part + (size_t)warp * D + (i * 32 + lane) * 4) = acc[i];
    __syncthreads();
    for (int j = tid * 4; j < D; j += 256 * 4) {
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const float4 v = *reinterpret_cast<const float4*>(s_part + (size_t)w * D + j);
        t.x += v.x, t.y += v.y, t.z += v.z, t.w += v.w;
      }
      const float ps = a.pgrad_scale;
      red_add_f32x4(dst + j, make_float4(t.x * ps, t.y * ps, t.z * ps, t.w * ps));
    }
  };
  flush(acc_g, a.dgamma);
  flush(acc_b, a.dbeta);
  flush(acc_c, a.colsum);
}

// Parameter gradients only (no dy requested): a pure column reduction, no per-row statistics of the gradient are needed.
// Thread = one column, block = 256 columns x kRowsPerBlock rows.
constexpr int kLnParamRows = 16;  // all 2 x 16 loads of a thread are issued before the first use (the loop is fully unrolled)
__global__ void __launch_bounds__(256) layernorm_bwd_params_kernel(const LnBwdArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  const int jj = blockIdx.x * 256 + threadIdx.x;
  const bool in = jj < a.d;         // threads past the row end stay in the loop: the Philox words travel by warp shuffle
  const int j = in ? jj : a.d - 1;  // (their loads hit a valid column, their sums are dropped)
  const int r0 = blockIdx.y * kLnParamRows;
  const int r1 = min(a.rows, r0 + kLnParamRows);
  float ag = 0.f, ab = 0.f;
#pragma unroll
  for (int rr = 0; rr < kLnParamRows; ++rr) {
    const int r = r0 + rr;
    if (r >= r1) break;  // warp-uniform
    float dj = __ldg(a.dout + (size_t)r * a.ld_dout + j);
    if (a.dout_mul) dj *= __ldg(a.dout_mul + (size_t)r * a.d + j);
    else if (drop.on) {  // the eight threads of an aligned column group share ONE Philox call (thread = column here)
      uint4 blk = make_uint4(0u, 0u, 0u, 0u);
      if ((threadIdx.x & 7) == 0) blk = drop_block(drop, (unsigned int)r, (unsigned int)(jj >> 3));
      const int src = (threadIdx.x & 31) & ~7;
      blk.x = __shfl_sync(0xffffffffu, blk.x, src);
      blk.y = __shfl_sync(0xffffffffu, blk.y, src);
      blk.z = __shfl_sync(0xffffffffu, blk.z, src);
      blk.w = __shfl_sync(0xffffffffu, blk.w, src);
      dj *= drop_pick(drop, blk, (unsigned int)(j & 7));
    }
    const float yv = a.y16 ? ld16(__ldg(a.y16 + (size_t)r * a.ld_y + j), a.y_fmt) : __ldg(a.y + (size_t)r * a.ld_y + j);
    const float xh = (yv - __ldg(a.mean + r)) * __ldg(a.rstd + r);
    ag += dj * xh;
    ab += dj;
  }
  if (in && a.dgamma) atomicAdd(a.dgamma + j, ag * a.pgrad_scale);
  if (in && a.dbeta) atomicAdd(a.dbeta + j, ab * a.pgrad_scale);
}

int launch_layernorm_bwd(const LnBwdArgs& a, cudaStream_t stream, int* kernel_used) {
  if (a.rows <= 0) return 0;
  if (a.dy32 == nullptr && a.dbr16 == nullptr) {
    if (kernel_used) *kernel_used = LNB_PARAMS;
    launch_k(layernorm_bwd_params_kernel, dim3(dim3((a.d + 255) / 256, (a.rows + kLnParamRows - 1) / kLnParamRows)), dim3(256), 0, stream, a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) set_error("layernorm_bwd launch failed: %s", cudaGetErrorString(e));
    return (int)e;
  }
  if (a.y16 != nullptr) {
    set_error("layernorm_bwd: a 16-bit LayerNorm input is only supported for the first projector layer (parameter gradients only)");
    return (int)cudaErrorInvalidValue;
  }
  static int max_blocks = 0;  // 4 blocks per SM by default; each block keeps register partials over its rows (UNIVTG_LNB_GRID overrides)
  if (max_blocks == 0) {
    const char* e = getenv("UNIVTG_LNB_GRID");
    max_blocks = (e != nullptr && atoi(e) > 0) ? atoi(e) : 592;
  }
  const int grid = a.rows < max_blocks ? a.rows : max_blocks;
  const bool vec = a.d % 4 == 0 && a.ld_dout % 4 == 0 && a.ld_y % 4 == 0 && (!a.dbr16 || a.ld16 % 4 == 0) &&
                   (((uintptr_t)a.dout | (uintptr_t)a.y | (uintptr_t)a.gamma | (uintptr_t)a.dy32 | (uintptr_t)a.dout_mul) & 15) == 0 &&
                   (((uintptr_t)a.dgamma | (uintptr_t)a.dbeta | (uintptr_t)a.colsum) & 15) == 0 && ((uintptr_t)a.dbr16 & 7) == 0;
  // warp-per-row kernel: d in {256, 512, 1024}, no K padding in the 16-bit output
  static int use_warp = -1;
  if (use_warp < 0) {
    const char* e = getenv("UNIVTG_LNB_WARP");
    use_warp = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  const bool warp_ok = use_warp && vec && (a.d == 256 || a.d == 512 || a.d == 1024) && (!a.dbr16 || a.ld16 == a.d);
  if (warp_ok) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int wgrid = (a.rows + 7) / 8;
    if (wgrid > sms) wgrid = sms;  // one 8-warp block per SM (253 registers per thread at d = 1024): a single wave
    const size_t smem = (size_t)8 * a.d * sizeof(float);
    if (a.d == 1024) launch_k(layernorm_bwd_warp_kernel<8>, dim3(wgrid), dim3(256), smem, stream, a);
    else if (a.d == 512) launch_k(layernorm_bwd_warp_kernel<4>, dim3(wgrid), dim3(256), smem, stream, a);
    else launch_k(layernorm_bwd_warp_kernel<2>, dim3(wgrid), dim3(256), smem, stream, a);
    if (kernel_used) *kernel_used = a.d == 1024 ? LNB_WARP8 : (a.d == 512 ? LNB_WARP4 : LNB_WARP2);
  } else if (vec && a.d <= 512) {
    launch_k(layernorm_bwd_vec_kernel<1>, dim3(grid), dim3(128), 0, stream, a);
    if (kernel_used) *kernel_used = LNB_VEC1;
  } else if (vec && a.d <= 1024) {
    launch_k(layernorm_bwd_vec_kernel<2>, dim3(grid), dim3(128), 0, stream, a);
    if (kernel_used) *kernel_used = LNB_VEC2;
  } else if (a.d <= 128 * 8) {
    launch_k(layernorm_bwd_kernel<8>, dim3(grid), dim3(128), 0, stream, a);
    if (kernel_used) *kernel_used = LNB_ROW8;
  } else if (a.d <= 128 * 24) {
    launch_k(layernorm_bwd_kernel<24>, dim3(grid), dim3(128), 0, stream, a);
    if (kernel_used) *kernel_used = LNB_ROW24;
  } else {
    set_error("layernorm_bwd: d %d > 3072 not supported", a.d);
    return (int)cudaErrorInvalidValue;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("layernorm_bwd launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// fp32 -> 16-bit conversion with optional column sums.  Block = 256 threads x 32 rows; thread = 4 columns.
// ------------------------------------------------------------------------------------------------
// text-row index of stream row r for the compact copy (TxtRows), or -1
__device__ __forceinline__ long long txt_row(const TxtRows& t, int r) {
  const int b = r / t.L, l = r - b * t.L;
  return l >= t.Lv ? (long long)b * (t.L - t.Lv) + (l - t.Lv) : -1;
}

template <bool TXT>
__global__ void __launch_bounds__(256) cvt16_colsum_kernel(const float* __restrict__ in32, int ld_in, uint16_t* __restrict__ out16,
                                                          int ld_out, int rows, int cols, int fmt, float* __restrict__ colsum, float cscale,
                                                          const TxtRows txt) {
  pdl_prologue();
  const int c = (blockIdx.x * 256 + threadIdx.x) * 4;
  if (c >= cols) return;
  const int r0 = blockIdx.y * 32;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = r0; r < min(rows, r0 + 32); ++r) {
    const float4 v = *reinterpret_cast<const float4*>(in32 + (size_t)r * ld_in + c);
    const uint2 h = make_uint2(cvt16x2(v.x, v.y, fmt), cvt16x2(v.z, v.w, fmt));
    *reinterpret_cast<uint2*>(out16 + (size_t)r * ld_out + c) = h;
    if constexpr (TXT) {
      const long long tr = txt_row(txt, r);
      if (tr >= 0 && c < txt.txt_cols) *reinterpret_cast<uint2*>(txt.txt16 + tr * txt.txt_cols + c) = h;
    }
    s.x += v.x;
    s.y += v.y;
    s.z += v.z;
    s.w += v.w;
  }
  if (colsum) {
    atomicAdd(colsum + c, s.x * cscale);
    atomicAdd(colsum + c + 1, s.y * cscale);
    atomicAdd(colsum + c + 2, s.z * cscale);
    atomicAdd(colsum + c + 3, s.w * cscale);
  }
}

// dst[n][c][t] = src[t][n][c] for the 3 taps of a k=3 conv weight gradient: the wgrad GEMMs write tap-major planes with
// 256-bit stores, this pass interleaves them into the reference's [out, in, 3] parameter layout (12 contiguous bytes per thread).
__global__ void __launch_bounds__(256) tap_interleave_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t nc) {
  pdl_prologue();
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < nc; i += (size_t)gridDim.x * 256) {
    const float a = __ldg(src + i), b = __ldg(src + nc + i), c = __ldg(src + 2 * nc + i);
    float* o = dst + 3 * i;
    o[0] = a;
    o[1] = b;
    o[2] = c;
  }
}
int launch_tap_interleave(const float* src, float* dst, int N, int C, cudaStream_t stream) {
  const size_t nc = (size_t)N * C;
  size_t blocks = (nc + 255) / 256;
  if (blocks > 2368) blocks = 2368;
  launch_k(tap_interleave_kernel, dim3((unsigned)blocks), dim3(256), 0, stream, src, dst, nc);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("tap_interleave launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// colsum[c] += scale * sum_r in16[r, c]: column sums of a 16-bit matrix (bias gradient of a GEMM whose output gradient was
// written directly in 16-bit).  thread = 8 columns (128-bit loads), block = 1024 columns x 64 rows.
constexpr int kColsumRows = 16;  // rows per block: all 16 loads of a thread are in flight at once (the first version walked 64
                                 // rows four loads at a time and sat at 13 us for 21 MB - latency, not bandwidth)
template <bool TXT>
__global__ void __launch_bounds__(128) colsum16_kernel(const uint16_t* __restrict__ in16, int ld, int rows, int cols, int fmt,
                                                      float* __restrict__ colsum, float scale, const TxtRows txt) {
  pdl_prologue();
  const int c = (blockIdx.x * 128 + threadIdx.x) * 8;
  if (c >= cols) return;
  const int r0 = blockIdx.y * kColsumRows;
  uint4 q[kColsumRows];
#pragma unroll
  for (int k = 0; k < kColsumRows; ++k)
    q[k] = (r0 + k < rows) ? __ldg(reinterpret_cast<const uint4*>(in16 + (size_t)(r0 + k) * ld + c)) : make_uint4(0u, 0u, 0u, 0u);
  if constexpr (TXT) {
    if (c < txt.txt_cols) {
#pragma unroll
      for (int k = 0; k < kColsumRows; ++k) {
        const long long tr = r0 + k < rows ? txt_row(txt, r0 + k) : -1;
        if (tr >= 0) *reinterpret_cast<uint4*>(txt.txt16 + tr * txt.txt_cols + c) = q[k];
      }
    }
  }
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < kColsumRows; ++k) {
    const uint32_t w[4] = {q[k].x, q[k].y, q[k].z, q[k].w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      s[2 * i] += ld16((uint16_t)(w[i] & 0xffff), fmt);
      s[2 * i + 1] += ld16((uint16_t)(w[i] >> 16), fmt);
    }
  }
  red_add_f32x4(colsum + c, make_float4(s[0] * scale, s[1] * scale, s[2] * scale, s[3] * scale));
  red_add_f32x4(colsum + c + 4, make_float4(s[4] * scale, s[5] * scale, s[6] * scale, s[7] * scale));
}

int launch_colsum16(const uint16_t* in16, int ld, int rows, int cols, int fmt, float* colsum, float scale, cudaStream_t stream,
                    TxtRows txt) {
  if (cols % 8 != 0 || ld % 8 != 0 || (reinterpret_cast<uintptr_t>(in16) & 15) != 0 || (reinterpret_cast<uintptr_t>(colsum) & 15) != 0 ||
      (txt.txt16 && (txt.txt_cols % 8 != 0 || (reinterpret_cast<uintptr_t>(txt.txt16) & 15) != 0))) {
    set_error("colsum16: columns / leading dimension must be multiples of 8 and the pointers 16-byte aligned");
    return (int)cudaErrorInvalidValue;
  }
  const dim3 grid((cols / 8 + 127) / 128, (rows + kColsumRows - 1) / kColsumRows);
  if (txt.txt16) launch_k(colsum16_kernel<true>, grid, dim3(128), 0, stream, in16, ld, rows, cols, fmt, colsum, scale, txt);
  else launch_k(colsum16_kernel<false>, grid, dim3(128), 0, stream, in16, ld, rows, cols, fmt, colsum, scale, txt);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("colsum16 launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

int launch_cvt16_colsum(const float* in32, int ld_in, uint16_t* out16, int ld_out, int rows, int cols, int fmt, float* colsum,
                        float colsum_scale, cudaStream_t stream, TxtRows txt) {
  if (cols % 4 != 0 || ld_in % 4 != 0 || ld_out % 4 != 0 || (txt.txt16 && txt.txt_cols % 4 != 0)) {
    set_error("cvt16_colsum: dims must be multiples of 4");
    return (int)cudaErrorInvalidValue;
  }
  dim3 grid((cols / 4 + 255) / 256, (rows + 31) / 32);
  if (txt.txt16)
    launch_k(cvt16_colsum_kernel<true>, dim3(grid), dim3(256), 0, stream, in32, ld_in, out16, ld_out, rows, cols, fmt, colsum, colsum_scale, txt);
  else
    launch_k(cvt16_colsum_kernel<false>, dim3(grid), dim3(256), 0, stream, in32, ld_in, out16, ld_out, rows, cols, fmt, colsum, colsum_scale, txt);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("cvt16_colsum launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// delta[b,h,i] = rowsum(dO * O) per head.  One warp per token row.
// ------------------------------------------------------------------------------------------------
// vec = 1 (dh % 8 == 0, 16-byte aligned rows): a lane owns 8 consecutive channels per step (128-bit loads of dO and O), dh / 8
// consecutive lanes cover one head and reduce among themselves - the scalar version moved 2 bytes per lane and load.
__global__ void __launch_bounds__(256) attn_delta_kernel(const uint16_t* __restrict__ dO, int fmt_do, const uint16_t* __restrict__ O,
                                                        int fmt_o, float* __restrict__ delta, int B, int L, int H, int dh, int vec) {
  pdl_prologue();
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= B * L) return;
  const int b = row / L, i = row - b * L;
  const int d = H * dh;
  if (vec) {
    const int lph = dh / 8;  // lanes per head: 16 (dh 128), 8 (dh 64), 4 (dh 32)
    for (int base = 0; base < d; base += 256) {  // warp-uniform trip count: the shuffles below need every lane
      const int c0 = base + lane * 8;
      const bool in = c0 < d;
      const uint4 x = in ? __ldg(reinterpret_cast<const uint4*>(dO + (size_t)row * d + c0)) : make_uint4(0u, 0u, 0u, 0u);
      const uint4 y = in ? __ldg(reinterpret_cast<const uint4*>(O + (size_t)row * d + c0)) : make_uint4(0u, 0u, 0u, 0u);
      const uint32_t xw[4] = {x.x, x.y, x.z, x.w}, yw[4] = {y.x, y.y, y.z, y.w};
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        s += ld16((uint16_t)(xw[k] & 0xffff), fmt_do) * ld16((uint16_t)(yw[k] & 0xffff), fmt_o) +
             ld16((uint16_t)(xw[k] >> 16), fmt_do) * ld16((uint16_t)(yw[k] >> 16), fmt_o);
      for (int o = lph >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (in && (lane & (lph - 1)) == 0) delta[((size_t)b * H + c0 / dh) * L + i] = s;
    }
    return;
  }
  for (int h = 0; h < H; ++h) {
    float s = 0.f;
    for (int c = lane; c < dh; c += 32) {
      const size_t idx = (size_t)row * d + h * dh + c;
      s += ld16(dO[idx], fmt_do) * ld16(O[idx], fmt_o);
    }
    s = warp_sum(s);
    if (lane == 0) delta[((size_t)b * H + h) * L + i] = s;
  }
}

int launch_attn_delta(const uint16_t* dO, int fmt_do, const uint16_t* O, int fmt_o, float* delta, int B, int L, int H, int dh,
                      cudaStream_t stream, int* vec_used) {
  const int rows = B * L;
  const int d = H * dh;
  // vector path: 8 channels per lane, 2^k lanes per head, every 256-channel step of a warp covers whole heads
  const int vec = (dh % 8 == 0) && ((dh / 8) & (dh / 8 - 1)) == 0 && dh <= 256 && (d % 8 == 0) && (256 % dh == 0 || dh == 256) &&
                  ((reinterpret_cast<uintptr_t>(dO) | reinterpret_cast<uintptr_t>(O)) & 15) == 0;
  if (vec_used) *vec_used = vec;
  launch_k(attn_delta_kernel, dim3((rows * 32 + 255) / 256), dim3(256), 0, stream, dO, fmt_do, O, fmt_o, delta, B, L, H, dh, vec ? 1 : 0);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("attn_delta launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// SIMT attention backward (any head size).  One warp per (b, h, query i); dK / dV / dQ accumulate atomically in fp32.
// ------------------------------------------------------------------------------------------------
// DROP = 1: the forward's attention dropout m (attn_drop_mul1, one Philox call per element): dV takes p m, dS = p (m dp - delta).
template <int DROP>
__global__ void __launch_bounds__(128) attention_bwd_simt_kernel(const AttnBwdArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  extern __shared__ float s_buf[];  // [4 warps][2][L]: p and ds
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * 4 + warp;
  if (gw >= a.B * a.H * a.L) return;
  const int i = gw % a.L;
  const int h = (gw / a.L) % a.H;
  const int b = gw / (a.L * a.H);
  float* p_s = s_buf + (size_t)warp * 2 * a.L;
  float* ds_s = p_s + a.L;
  const size_t ld = (size_t)3 * a.d;
  const uint16_t* qrow = a.qkv + ((size_t)b * a.L + i) * ld + h * a.dh;
  const uint16_t* dorow = a.dO + ((size_t)b * a.L + i) * a.d + h * a.dh;
  const float lse = a.lse[((size_t)b * a.H + h) * a.L + i];
  const float dlt = a.delta[((size_t)b * a.H + h) * a.L + i];
  for (int j = lane; j < a.L; j += 32) {
    float p = 0.f, ds = 0.f;
    if (a.key_mask[(size_t)b * a.L + j] != 0.f) {
      const uint16_t* krow = a.qkv + ((size_t)b * a.L + j) * ld + a.d + h * a.dh;
      const uint16_t* vrow = a.qkv + ((size_t)b * a.L + j) * ld + 2 * a.d + h * a.dh;
      float s = 0.f, dp = 0.f;
      for (int c = 0; c < a.dh; ++c) {
        s += ld16(qrow[c], a.fmt_act) * ld16(krow[c], a.fmt_act);
        dp += ld16(dorow[c], a.fmt_grad) * ld16(vrow[c], a.fmt_act);
      }
      p = expf(s * a.scale - lse);
      if constexpr (DROP != 0) {
        const float m = attn_drop_mul1(drop, (unsigned int)(b * a.H + h), (unsigned int)i, (unsigned int)j);
        ds = p * (m * dp - dlt) * a.scale;
        p *= m;
      } else {
        ds = p * (dp - dlt) * a.scale;
      }
    }
    p_s[j] = p;
    ds_s[j] = ds;
  }
  __syncwarp();
  for (int c = lane; c < a.dh; c += 32) {
    const float qc = ld16(qrow[c], a.fmt_act);
    const float doc = ld16(dorow[c], a.fmt_grad);
    float dq = 0.f;
    for (int j = 0; j < a.L; ++j) {
      const float ds = ds_s[j], p = p_s[j];
      if (p == 0.f && ds == 0.f) continue;
      const size_t kbase = ((size_t)b * a.L + j) * ld;
      dq += ds * ld16(a.qkv[kbase + a.d + h * a.dh + c], a.fmt_act);
      atomicAdd(a.dqkv32 + kbase + a.d + h * a.dh + c, ds * qc);
      atomicAdd(a.dqkv32 + kbase + 2 * a.d + h * a.dh + c, p * doc);
    }
    atomicAdd(a.dqkv32 + ((size_t)b * a.L + i) * ld + h * a.dh + c, dq);
  }
}

int launch_attention_bwd_simt(const AttnBwdArgs& a, cudaStream_t stream, int* kernel_used) {
  const int warps = a.B * a.H * a.L;
  const size_t smem = attention_bwd_simt_smem(a.L);
  auto kern = a.drop.on ? attention_bwd_simt_kernel<1> : attention_bwd_simt_kernel<0>;
  if (kernel_used) *kernel_used = 8 + (a.drop.on ? 1 : 0);
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("attention_bwd_simt smem %zu: %s", smem, cudaGetErrorString(e));
      return (int)e;
    }
  }
  launch_k(kern, dim3((warps + 3) / 4), dim3(128), smem, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("attention_bwd_simt launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// Heads, last conv layer backward.
//   z_o[m] = b_o + sum_t sum_c W[o, c, t] h[m + t - 1, c];  pred = (+-) sigmoid(z)
// kernel 1: dz (pre-sigmoid gradients) per clip, conv layout, separators zero
// kernel 2: dh[m', c] = relu'(h[m', c]) * sum_t sum_o dz_o[m' - t + 1] W[o, c, t]   (+ column sums)
// kernel 3: dW[o, c, t] = sum_m dz_o[m] h[m + t - 1, c],  db[o] = sum_m dz_o[m]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) head_dz_kernel(const HeadFinalBwdArgs a) {
  pdl_prologue();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int rows = a.B * (a.Lv + 1) + 2;
  if (idx >= rows) return;
  float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
  const int m = idx - 1;  // logical conv row
  if (m >= 0 && m < a.B * (a.Lv + 1)) {
    const int b = m / (a.Lv + 1), l = m - b * (a.Lv + 1);
    if (l < a.Lv) {
      const size_t k = (size_t)b * a.Lv + l;
      const float pc = a.pred_logits[k];
      const float s0 = -a.pred_spans[2 * k];  // sigmoid value of the left offset (stored negated)
      const float s1 = a.pred_spans[2 * k + 1];
      out.x = a.in_scale * a.g_logits[k] * pc * (1.f - pc);
      out.y = -a.in_scale * a.g_spans[2 * k] * s0 * (1.f - s0);
      out.z = a.in_scale * a.g_spans[2 * k + 1] * s1 * (1.f - s1);
    }
  }
  *reinterpret_cast<float4*>(a.dz + (size_t)idx * 4) = out;
}

__global__ void __launch_bounds__(256) head_dh_kernel(const HeadFinalBwdArgs a) {
  pdl_prologue();
  // one warp per buffer row (1 .. B*(Lv+1)); lanes over channels
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int Mh = a.B * (a.Lv + 1);
  if (gw >= Mh) return;
  const size_t row = (size_t)gw + 1;  // buffer row of logical row m' = gw
  const int l = gw % (a.Lv + 1);
  const bool sep = (l == a.Lv);
  // dz of logical rows m' - t + 1 for t = 0, 1, 2  -> buffer rows row + 1 - t
  float dzc[3], dz0[3], dz1[3];
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    const float4 v = *reinterpret_cast<const float4*>(a.dz + (row + 1 - t) * 4);
    dzc[t] = v.x;
    dz0[t] = v.y;
    dz1[t] = v.z;
  }
  for (int c = lane * 2; c < a.d; c += 64) {
    float gc[2] = {0.f, 0.f}, gs[2] = {0.f, 0.f};
    if (!sep) {
#pragma unroll
      for (int t = 0; t < 3; ++t) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          gc[e] += dzc[t] * a.w_cls[(size_t)t * a.d + c + e];
          gs[e] += dz0[t] * a.w_span[(size_t)t * a.d + c + e] + dz1[t] * a.w_span[(size_t)(3 + t) * a.d + c + e];
        }
      }
      const uint32_t hc = *reinterpret_cast<const uint32_t*>(a.h_cls + row * a.d + c);
      const uint32_t hs = *reinterpret_cast<const uint32_t*>(a.h_span + row * a.d + c);
      if (!pos16((uint16_t)(hc & 0xffff))) gc[0] = 0.f;
      if (!pos16((uint16_t)(hc >> 16))) gc[1] = 0.f;
      if (!pos16((uint16_t)(hs & 0xffff))) gs[0] = 0.f;
      if (!pos16((uint16_t)(hs >> 16))) gs[1] = 0.f;
    }
    *reinterpret_cast<uint32_t*>(a.dh_cls + row * a.d + c) = cvt16x2(gc[0], gc[1], a.fmt_grad);
    *reinterpret_cast<uint32_t*>(a.dh_span + row * a.d + c) = cvt16x2(gs[0], gs[1], a.fmt_grad);
  }
}

// Weight / bias gradients of the heads' last conv layer and the column sums of dh (bias gradient of the layer before).
// thread = 8 consecutive channels (128-bit loads), block = 1024 channels x a slab of kHeadDwRows logical rows; the three tap
// rows (m-1, m, m+1) slide through registers so every activation row is read once.
constexpr int kHeadDwRows = 32;
__device__ __forceinline__ void ld8(const uint16_t* p, int fmt, float (&v)[8]) {
  const uint4 q = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[2 * i] = ld16((uint16_t)(w[i] & 0xffff), fmt);
    v[2 * i + 1] = ld16((uint16_t)(w[i] >> 16), fmt);
  }
}
__global__ void __launch_bounds__(128) head_dw_kernel(const HeadFinalBwdArgs a) {
  pdl_prologue();
  const int c = (blockIdx.x * 128 + threadIdx.x) * 8;
  const int Mh = a.B * (a.Lv + 1);
  const int m0 = blockIdx.y * kHeadDwRows;
  const int m1 = min(Mh, m0 + kHeadDwRows);
  if (c < a.d) {
    float wc[3][8], w0[3][8], w1[3][8], cs_c[8], cs_s[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      cs_c[j] = cs_s[j] = 0.f;
#pragma unroll
      for (int t = 0; t < 3; ++t) wc[t][j] = w0[t][j] = w1[t][j] = 0.f;
    }
    float pc[8], cc[8], nc[8], ps[8], cu[8], ns[8];  // previous / current / next activation row of both heads
    ld8(a.h_cls + (size_t)m0 * a.d + c, a.fmt_act, pc);
    ld8(a.h_span + (size_t)m0 * a.d + c, a.fmt_act, ps);
    ld8(a.h_cls + (size_t)(m0 + 1) * a.d + c, a.fmt_act, cc);
    ld8(a.h_span + (size_t)(m0 + 1) * a.d + c, a.fmt_act, cu);
    for (int m = m0; m < m1; ++m) {
      const size_t row = (size_t)m + 1;
      ld8(a.h_cls + (row + 1) * a.d + c, a.fmt_act, nc);
      ld8(a.h_span + (row + 1) * a.d + c, a.fmt_act, ns);
      const float4 dz = *reinterpret_cast<const float4*>(a.dz + row * 4);
      if (a.cs_cls) {
        float gc[8], gs[8];
        ld8(a.dh_cls + row * a.d + c, a.fmt_grad, gc);
        ld8(a.dh_span + row * a.d + c, a.fmt_grad, gs);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          cs_c[j] += gc[j];
          cs_s[j] += gs[j];
        }
      }
      if (dz.x != 0.f || dz.y != 0.f || dz.z != 0.f) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          wc[0][j] += dz.x * pc[j];
          wc[1][j] += dz.x * cc[j];
          wc[2][j] += dz.x * nc[j];
          w0[0][j] += dz.y * ps[j];
          w0[1][j] += dz.y * cu[j];
          w0[2][j] += dz.y * ns[j];
          w1[0][j] += dz.z * ps[j];
          w1[1][j] += dz.z * cu[j];
          w1[2][j] += dz.z * ns[j];
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        pc[j] = cc[j];
        cc[j] = nc[j];
        ps[j] = cu[j];
        cu[j] = ns[j];
      }
    }
    // this thread's 8 channels x 3 taps are 24 consecutive floats of each [.., d, 3] weight gradient: six 128-bit reductions
    const float gsc = a.pgrad_scale;
    float* dsts[3] = {a.gw_cls + (size_t)c * 3, a.gw_span + (size_t)c * 3, a.gw_span + ((size_t)a.d + c) * 3};
#pragma unroll
    for (int w = 0; w < 3; ++w) {
      float flat[24];
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int t = 0; t < 3; ++t) flat[j * 3 + t] = (w == 0 ? wc[t][j] : (w == 1 ? w0[t][j] : w1[t][j])) * gsc;
#pragma unroll
      for (int q = 0; q < 6; ++q)
        red_add_f32x4(dsts[w] + 4 * q, make_float4(flat[4 * q], flat[4 * q + 1], flat[4 * q + 2], flat[4 * q + 3]));
    }
    if (a.cs_cls) {
      red_add_f32x4(a.cs_cls + c, make_float4(cs_c[0] * gsc, cs_c[1] * gsc, cs_c[2] * gsc, cs_c[3] * gsc));
      red_add_f32x4(a.cs_cls + c + 4, make_float4(cs_c[4] * gsc, cs_c[5] * gsc, cs_c[6] * gsc, cs_c[7] * gsc));
      red_add_f32x4(a.cs_span + c, make_float4(cs_s[0] * gsc, cs_s[1] * gsc, cs_s[2] * gsc, cs_s[3] * gsc));
      red_add_f32x4(a.cs_span + c + 4, make_float4(cs_s[4] * gsc, cs_s[5] * gsc, cs_s[6] * gsc, cs_s[7] * gsc));
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {  // bias gradients: sum of dz over this slab
    float bc = 0.f, b0 = 0.f, b1 = 0.f;
    for (int m = m0; m < m1; ++m) {
      const float4 dz = *reinterpret_cast<const float4*>(a.dz + ((size_t)m + 1) * 4);
      bc += dz.x;
      b0 += dz.y;
      b1 += dz.z;
    }
    atomicAdd(a.gb_cls, bc * a.pgrad_scale);
    atomicAdd(a.gb_span, b0 * a.pgrad_scale);
    atomicAdd(a.gb_span + 1, b1 * a.pgrad_scale);
  }
}

int launch_head_final_bwd(const HeadFinalBwdArgs& a, cudaStream_t stream) {
  const int Mh = a.B * (a.Lv + 1);
  launch_k(head_dz_kernel, dim3((Mh + 2 + 255) / 256), dim3(256), 0, stream, a);
  launch_k(head_dh_kernel, dim3((Mh * 32 + 255) / 256), dim3(256), 0, stream, a);
  launch_k(head_dw_kernel, dim3((a.d + 1023) / 1024, (Mh + kHeadDwRows - 1) / kHeadDwRows), dim3(128), 0, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("head_final_bwd launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// Weighted pool backward.  pooled = sum_l alpha_l x_l, alpha = softmax(x . w + mask bias).  One CTA per sample.
//   dalpha_l = g . x_l;  dlogit_l = alpha_l (dalpha_l - sum_k alpha_k dalpha_k)
//   dx_l = alpha_l g + dlogit_l w;  dw += sum_l dlogit_l x_l
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pool_bwd_kernel(const PoolBwdArgs a) {
  pdl_prologue();
  extern __shared__ float sm[];
  float* s_da = sm;              // [Lt] dalpha, then dlogit
  __shared__ float s_dot;
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const float* xt = a.x_txt + (size_t)b * a.Lt * a.d;
  const float* g = a.g_pooled + (size_t)b * a.d;
  const float* al = a.alpha + (size_t)b * a.Lt;
  for (int l = warp; l < a.Lt; l += nw) {
    float s = 0.f;
    for (int j = lane; j < a.d; j += 32) s += g[j] * xt[(size_t)l * a.d + j];
    s = warp_sum(s);
    if (lane == 0) s_da[l] = s;
  }
  __syncthreads();
  if (warp == 0) {
    float s = 0.f;
    for (int l = lane; l < a.Lt; l += 32) s += al[l] * s_da[l];
    s = warp_sum(s);
    if (lane == 0) s_dot = s;
  }
  __syncthreads();
  const float dot = s_dot;
  for (int l = threadIdx.x; l < a.Lt; l += blockDim.x) s_da[l] = al[l] * (s_da[l] - dot);
  __syncthreads();
  for (int j = threadIdx.x; j < a.d; j += blockDim.x) {
    const float gj = g[j], wj = a.w[j];
    float dw = 0.f;
    for (int l = 0; l < a.Lt; ++l) {
      const float dl = s_da[l];
      a.dx_txt[((size_t)b * a.Lt + l) * a.d + j] = (al[l] * gj + dl * wj) * a.out_scale;
      dw += dl * xt[(size_t)l * a.d + j];
    }
    atomicAdd(a.gw + j, dw);
  }
}

int launch_pool_bwd(const PoolBwdArgs& a, cudaStream_t stream) {
  launch_k(pool_bwd_kernel, dim3(a.B), dim3(256), (size_t)a.Lt * sizeof(float), stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("pool_bwd launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// Projector-output gradient assembly: rows of one modality gathered from the stream gradient + the direct
// (saliency-loss) gradient, emitted as a 16-bit GEMM operand with column sums.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) stream_gather_kernel(const float* __restrict__ dx, int L, int off, const float* __restrict__ extra,
                                                           float extra_scale, uint16_t* __restrict__ out16,
                                                           float* __restrict__ colsum, float cscale, int B, int Ls, int d, int fmt) {
  pdl_prologue();
  const int c = (blockIdx.x * 256 + threadIdx.x) * 4;
  if (c >= d) return;
  const int r0 = blockIdx.y * 32;
  const int rows = B * Ls;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = r0; r < min(rows, r0 + 32); ++r) {
    const int b = r / Ls, l = r - b * Ls;
    float4 v = *reinterpret_cast<const float4*>(dx + ((size_t)b * L + off + l) * d + c);
    if (extra) {
      const float4 e = *reinterpret_cast<const float4*>(extra + (size_t)r * d + c);
      v.x += e.x * extra_scale;
      v.y += e.y * extra_scale;
      v.z += e.z * extra_scale;
      v.w += e.w * extra_scale;
    }
    *reinterpret_cast<uint2*>(out16 + (size_t)r * d + c) = make_uint2(cvt16x2(v.x, v.y, fmt), cvt16x2(v.z, v.w, fmt));
    s.x += v.x;
    s.y += v.y;
    s.z += v.z;
    s.w += v.w;
  }
  if (colsum) {
    atomicAdd(colsum + c, s.x * cscale);
    atomicAdd(colsum + c + 1, s.y * cscale);
    atomicAdd(colsum + c + 2, s.z * cscale);
    atomicAdd(colsum + c + 3, s.w * cscale);
  }
}

int launch_stream_gather(const float* dx_stream, int L, int off, const float* extra, float extra_scale, uint16_t* out16,
                         float* colsum, float colsum_scale, int B, int Ls, int d, int fmt, cudaStream_t stream) {
  dim3 grid((d / 4 + 255) / 256, (B * Ls + 31) / 32);
  launch_k(stream_gather_kernel, dim3(grid), dim3(256), 0, stream, dx_stream, L, off, extra, extra_scale, out16, colsum, colsum_scale, B, Ls, d, fmt);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("stream_gather launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}


// ------------------------------------------------------------------------------------------------
// Learned text positions backward (TxtPosBwdArgs, backward.h).  One 128-thread CTA per position l; thread owns columns
// tid + 128 i.  The position-table row l is this CTA's alone: no atomics for dtable.
// ------------------------------------------------------------------------------------------------
template <int EPT>
__global__ void __launch_bounds__(128) txt_pos_bwd_kernel(const TxtPosBwdArgs a) {
  pdl_prologue();
  const DropSpec drop = drop_resolve(a.drop);
  __shared__ float s_red[2][2][4];  // [parity of b][sum g, sum g * xhat][warp]
  const int l = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* P = a.table + (size_t)l * a.d;
  float acc_p[EPT], acc_g[EPT], acc_b[EPT], pv[EPT], gam[EPT];
#pragma unroll
  for (int i = 0; i < EPT; ++i) {
    const int j = tid + 128 * i;
    acc_p[i] = acc_g[i] = acc_b[i] = 0.f;
    pv[i] = j < a.d ? P[j] : 0.f;
    gam[i] = j < a.d ? a.gamma[j] : 0.f;
  }
  for (int b = 0; b < a.B; ++b) {
    const size_t r = (size_t)b * a.Lt + l;
    const float mean = a.mean[r], rstd = a.rstd[r];
    float g[EPT], xh[EPT];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const int j = tid + 128 * i;
      g[i] = xh[i] = 0.f;
      if (j < a.d) {
        float go = a.dpos[r * a.d + j];
        if (a.mul32) go *= a.mul32[r * a.d + j];
        else if (drop.on) go *= drop_mul1(drop, (unsigned int)r, (unsigned int)j);
        xh[i] = (a.xt[r * a.d + j] + pv[i] - mean) * rstd;
        acc_g[i] += go * xh[i];
        acc_b[i] += go;
        g[i] = go * gam[i];
        s1 += g[i];
        s2 += g[i] * xh[i];
      }
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (lane == 0) {
      s_red[b & 1][0][warp] = s1;
      s_red[b & 1][1][warp] = s2;
    }
    __syncthreads();  // (double-buffered by the parity of b: one barrier per sample)
    const float m1 = (s_red[b & 1][0][0] + s_red[b & 1][0][1] + s_red[b & 1][0][2] + s_red[b & 1][0][3]) / (float)a.d;
    const float m2 = (s_red[b & 1][1][0] + s_red[b & 1][1][1] + s_red[b & 1][1][2] + s_red[b & 1][1][3]) / (float)a.d;
    float* dxr = a.dx + ((size_t)b * a.L + a.Lv + l) * a.d;
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const int j = tid + 128 * i;
      if (j < a.d) {
        const float du = rstd * (g[i] - m1 - xh[i] * m2);
        acc_p[i] += du;
        dxr[j] += du;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < EPT; ++i) {
    const int j = tid + 128 * i;
    if (j < a.d) {
      a.dtable[(size_t)l * a.d + j] = acc_p[i] * a.pgrad_scale;
      atomicAdd(a.dgamma + j, acc_g[i] * a.pgrad_scale);
      atomicAdd(a.dbeta + j, acc_b[i] * a.pgrad_scale);
    }
  }
}

int launch_txt_pos_bwd(const TxtPosBwdArgs& a, cudaStream_t stream) {
  if (a.d > 128 * 8) {
    set_error("txt_pos_bwd: hidden_dim %d > 1024 not supported", a.d);
    return (int)cudaErrorInvalidValue;
  }
  launch_k(txt_pos_bwd_kernel<8>, dim3(a.Lt), dim3(128), 0, stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("txt_pos_bwd launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

}  // namespace uv
