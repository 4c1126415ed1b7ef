// Parameter update of the reference's training loop over ONE flat fp32 buffer (main/train_vlp_ddp.py:66-68, main/train_mr.py:64-66,
// optimizer built at main/config.py:350): total-norm gradient clipping (torch.nn.utils.clip_grad_norm_, L2) followed by
// torch.optim.AdamW (decoupled weight decay, bias-corrected, no amsgrad).  Two launches: sum of squares, then the update with
// the clip coefficient computed on the device - no host round trip.  HBM-bound: 16 B read + 12 B written per parameter.
#include <math.h>
#include <stdint.h>

#include "../../include/univtg_b200.h"
#include "kernels.h"
#include "ptx.cuh"

namespace uv {
namespace {

// Per-block partial sums of squares, written to partial[blockIdx.x] (no atomics): the update kernel adds them in a fixed order, so
// the gradient norm - and with it the clip factor and every updated weight - is bit-reproducible and bit-identical on every
// data-parallel rank (an atomicAdd accumulation differs in the last bits from GPU to GPU, and the replicas then drift apart).
__device__ __forceinline__ void sumsq_body(const float* __restrict__ g, size_t n4, float* __restrict__ partial) {
  __shared__ float s_red[8];
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float s = 0.f;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n4; i += (size_t)gridDim.x * 256) {
    const float4 v = __ldg(g4 + i);
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s_red[i];
    partial[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, size_t n4, float* __restrict__ partial) {
  pdl_prologue();
  sumsq_body(g, n4, partial);
}
// univtg_adamw_step_dev: also stages the step of this update, *step_dev + 1, in scratch[3] (the update kernel reads it there and
// block 0 writes it back to step_dev, so no block of the update reads step_dev while another one writes it)
__global__ void __launch_bounds__(256) sumsq_dev_kernel(const float* __restrict__ g, size_t n4, float* __restrict__ scratch,
                                                        const int32_t* __restrict__ step_dev) {
  pdl_prologue();
  if (blockIdx.x == 0 && threadIdx.x == 0) reinterpret_cast<int32_t*>(scratch)[3] = *step_dev + 1;
  sumsq_body(g, n4, scratch + 4);
}

// fixed-order total of the per-block partials (every block of the update kernel computes the same value)
__device__ __forceinline__ float ordered_total(const float* __restrict__ partial, int n, float* s_red) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) s += partial[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = s;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < 8; ++i) t += s_red[i];
  __syncthreads();
  return t;
}

struct AdamArgs {
  float* p;
  const float* g;
  float* m;
  float* v;
  size_t n4;
  float lr, beta1, beta2, eps, wd, bc1, bc2_sqrt, max_norm;
  float* scratch;  // [1] = total norm (out), [2] = 1 when the step was skipped (non-finite gradients), [3] = int32 step staged by
                   // sumsq_dev_kernel (device-state variant only), [4 ..) = per-block partial sums (in)
  int n_partial;
  float* g_out;    // clipped gradients written back (clip_grad_norm_ scales .grad in place) or null
};

// 16-bit operand copy of the four freshly updated parameters at flat float4 index i (see PackSeg)
__device__ __forceinline__ void pack_updated(const PackSegTable& t, size_t i, const float4& p) {
  int lo = 0, hi = t.n;  // first segment with start4 > i
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((size_t)t.s[mid].start4 <= i) lo = mid + 1;
    else hi = mid;
  }
  if (lo == 0) return;
  const PackSeg& sg = t.s[lo - 1];
  if (i >= (size_t)sg.end4) return;
  const size_t e = (i - (size_t)sg.start4) * 4;
  uint16_t* dst = reinterpret_cast<uint16_t*>(sg.dst);
  const float v[4] = {p.x, p.y, p.z, p.w};
  if (sg.kind == 0) {
    const size_t r = e / (size_t)sg.cols;
    const int c = (int)(e - r * (size_t)sg.cols);
    if ((sg.cols & 3) == 0) {  // four columns of one row, 8-byte aligned (ld % 4 == 0)
      *reinterpret_cast<uint2*>(dst + r * (size_t)sg.ld + c) = make_uint2(cvt16x2(p.x, p.y, t.fmt), cvt16x2(p.z, p.w, t.fmt));
    } else {
      size_t rr = r;
      int cc = c;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (rr < (size_t)sg.rows) dst[rr * (size_t)sg.ld + cc] = cvt16(v[q], t.fmt);
        if (++cc == sg.cols) {
          cc = 0;
          ++rr;
        }
      }
    }
  } else {
    const size_t C3 = (size_t)3 * sg.cols;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const size_t eq = e + q;
      const size_t n = eq / C3;
      const int rem = (int)(eq - n * C3);
      const int c = rem / 3, tap = rem - 3 * c;
      if (n < (size_t)sg.rows) dst[n * C3 + (size_t)tap * sg.cols + c] = cvt16(v[q], t.fmt);
    }
  }
}

// the update with (lr, bc1, bc2_sqrt) given; returns whether the step was skipped (the same answer in every block)
template <bool PACK>
__device__ __forceinline__ bool adamw_body(const AdamArgs& a, const float lr, const float bc1, const float bc2_sqrt,
                                           const PackSegTable& segs) {
  __shared__ float s_red[8];
  const float norm = sqrtf(ordered_total(a.scratch + 4, a.n_partial, s_red));
  float clip = 1.f;
  if (a.max_norm > 0.f) clip = fminf(a.max_norm / (norm + 1e-6f), 1.f);
  // fp16 loss-scaled backward: an overflow in a 16-bit gradient operand shows up as inf / NaN in the gradient buffer, hence in its
  // norm.  Such a step must leave weights and moments untouched (what torch.cuda.amp.GradScaler.step does); the caller reads
  // scratch[2] later (no synchronisation here) and backs the loss scale off.
  const bool skip = !isfinite(norm);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.scratch[1] = norm;
    a.scratch[2] = skip ? 1.f : 0.f;
  }
  if (skip) return true;
  float4* p4 = reinterpret_cast<float4*>(a.p);
  const float4* g4 = reinterpret_cast<const float4*>(a.g);
  float4* m4 = reinterpret_cast<float4*>(a.m);
  float4* v4 = reinterpret_cast<float4*>(a.v);
  const float decay = 1.f - lr * a.wd, step = lr / bc1, ob1 = 1.f - a.beta1, ob2 = 1.f - a.beta2;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < a.n4; i += (size_t)gridDim.x * 256) {
    float4 p = p4[i], g = __ldg(g4 + i), m = m4[i], v = v4[i];
#define UV_ADAM(c)                                         \
  g.c *= clip;                                             \
  p.c *= decay;                                            \
  m.c = fmaf(g.c - m.c, ob1, m.c);                         \
  v.c = fmaf(a.beta2, v.c, ob2 * g.c * g.c);               \
  p.c -= step * m.c / (sqrtf(v.c) / bc2_sqrt + a.eps);
    UV_ADAM(x) UV_ADAM(y) UV_ADAM(z) UV_ADAM(w)
#undef UV_ADAM
    p4[i] = p;
    m4[i] = m;
    v4[i] = v;
    if (PACK) pack_updated(segs, i, p);
    if (a.g_out) reinterpret_cast<float4*>(a.g_out)[i] = g;
  }
  return false;
}

template <bool PACK>
__global__ void __launch_bounds__(256) adamw_kernel(const AdamArgs a, const __grid_constant__ PackSegTable segs) {
  pdl_prologue();
  adamw_body<PACK>(a, a.lr, a.bc1, a.bc2_sqrt, segs);
}

// Device-state variant (CUDA-graph replay): lr from device memory, the step t staged in scratch[3] by sumsq_dev_kernel, and
// (bc1, bc2_sqrt) = table[2 (t - 1)], table[2 (t - 1) + 1], filled on the host with adamw_step_impl's own expressions, so the
// update is bit-identical to univtg_adamw_step at the same step.  Steps past the table reuse its last row.  t is written back to
// step_dev only when the step was not skipped.
struct AdamDevArgs {
  const float* lr;
  int32_t* step;
  const float* bc;
  int bc_len;
};
template <bool PACK>
__global__ void __launch_bounds__(256) adamw_dev_kernel(const AdamArgs a, const AdamDevArgs dv, const __grid_constant__ PackSegTable segs) {
  pdl_prologue();
  const int32_t t = reinterpret_cast<const int32_t*>(a.scratch)[3];
  const int r = (t < dv.bc_len ? (t > 1 ? t : 1) : dv.bc_len) - 1;
  const bool skip = adamw_body<PACK>(a, *dv.lr, dv.bc[2 * r], dv.bc[2 * r + 1], segs);
  if (!skip && blockIdx.x == 0 && threadIdx.x == 0) *dv.step = t;
}

}  // namespace
}  // namespace uv

namespace uv {
void adamw_bias_row(float beta1, float beta2, int32_t step, float* bc1, float* bc2_sqrt) {
  // the expressions of adamw_step_impl below: the device-state update reads exactly these floats from its table
  *bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  *bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
}

int adamw_step_impl(float* params, float* grads, float* exp_avg, float* exp_avg_sq, size_t n, float lr, float beta1, float beta2,
                    float eps, float weight_decay, int32_t step, float max_grad_norm, int32_t write_clipped_grads, float* scratch2,
                    const PackSegTable* segs, void* stream, const AdamDevState* dev) {
  using namespace uv;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (n == 0) return 0;
  if (n % 4 != 0 || (dev == nullptr && step < 1) ||
      ((((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq)) & 15) != 0 || scratch2 == nullptr) {
    set_error("univtg_adamw_step: buffers must be 16-byte aligned with n %% 4 == 0, step >= 1, scratch non-null");
    return (int)cudaErrorInvalidValue;
  }
  int dev_id = 0, sms = 132;
  cudaGetDevice(&dev_id);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev_id);
  const size_t n4 = n / 4;
  size_t blocks = (n4 + 255) / 256;
  if (blocks > (size_t)sms * 8) blocks = (size_t)sms * 8;
  if (blocks > UNIVTG_ADAMW_SCRATCH_FLOATS - 4) blocks = UNIVTG_ADAMW_SCRATCH_FLOATS - 4;
  if (dev) launch_k(sumsq_dev_kernel, dim3((unsigned)blocks), dim3(256), 0, st, grads, n4, scratch2, dev->step);
  else launch_k(sumsq_kernel, dim3((unsigned)blocks), dim3(256), 0, st, grads, n4, scratch2 + 4);
  AdamArgs a;
  a.p = params;
  a.g = grads;
  a.m = exp_avg;
  a.v = exp_avg_sq;
  a.n4 = n4;
  a.lr = lr;
  a.beta1 = beta1;
  a.beta2 = beta2;
  a.eps = eps;
  a.wd = weight_decay;
  if (dev) a.bc1 = a.bc2_sqrt = 1.f;  // (read from the table on the device)
  else adamw_bias_row(beta1, beta2, step, &a.bc1, &a.bc2_sqrt);
  a.max_norm = max_grad_norm;
  a.scratch = scratch2;
  a.n_partial = (int)blocks;
  a.g_out = write_clipped_grads ? grads : nullptr;
  PackSegTable none;
  none.n = 0;
  none.fmt = 0;
  const bool pack = segs != nullptr && segs->n > 0;
  if (dev) {
    const AdamDevArgs dv{dev->lr, dev->step, dev->bc_table, dev->table_len};
    if (pack) launch_k(adamw_dev_kernel<true>, dim3((unsigned)blocks), dim3(256), 0, st, a, dv, *segs);
    else launch_k(adamw_dev_kernel<false>, dim3((unsigned)blocks), dim3(256), 0, st, a, dv, none);
  } else if (pack) {
    launch_k(adamw_kernel<true>, dim3((unsigned)blocks), dim3(256), 0, st, a, *segs);
  } else {
    launch_k(adamw_kernel<false>, dim3((unsigned)blocks), dim3(256), 0, st, a, none);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_adamw_step launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}
}  // namespace uv
