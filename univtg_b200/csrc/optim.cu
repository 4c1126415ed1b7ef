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
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, size_t n4, float* __restrict__ partial) {
  pdl_prologue();
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
  float* scratch;  // [1] = total norm (out), [2] = 1 when the step was skipped (non-finite gradients), [4 ..) = per-block partial sums (in)
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

template <bool PACK>
__global__ void __launch_bounds__(256) adamw_kernel(const AdamArgs a, const __grid_constant__ PackSegTable segs) {
  pdl_prologue();
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
  if (skip) return;
  float4* p4 = reinterpret_cast<float4*>(a.p);
  const float4* g4 = reinterpret_cast<const float4*>(a.g);
  float4* m4 = reinterpret_cast<float4*>(a.m);
  float4* v4 = reinterpret_cast<float4*>(a.v);
  const float decay = 1.f - a.lr * a.wd, step = a.lr / a.bc1, ob1 = 1.f - a.beta1, ob2 = 1.f - a.beta2;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < a.n4; i += (size_t)gridDim.x * 256) {
    float4 p = p4[i], g = __ldg(g4 + i), m = m4[i], v = v4[i];
#define UV_ADAM(c)                                         \
  g.c *= clip;                                             \
  p.c *= decay;                                            \
  m.c = fmaf(g.c - m.c, ob1, m.c);                         \
  v.c = fmaf(a.beta2, v.c, ob2 * g.c * g.c);               \
  p.c -= step * m.c / (sqrtf(v.c) / a.bc2_sqrt + a.eps);
    UV_ADAM(x) UV_ADAM(y) UV_ADAM(z) UV_ADAM(w)
#undef UV_ADAM
    p4[i] = p;
    m4[i] = m;
    v4[i] = v;
    if (PACK) pack_updated(segs, i, p);
    if (a.g_out) reinterpret_cast<float4*>(a.g_out)[i] = g;
  }
}

}  // namespace
}  // namespace uv

namespace uv {
int adamw_step_impl(float* params, float* grads, float* exp_avg, float* exp_avg_sq, size_t n, float lr, float beta1, float beta2,
                    float eps, float weight_decay, int32_t step, float max_grad_norm, int32_t write_clipped_grads, float* scratch2,
                    const PackSegTable* segs, void* stream) {
  using namespace uv;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (n == 0) return 0;
  if (n % 4 != 0 || step < 1 || ((((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq)) & 15) != 0 ||
      scratch2 == nullptr) {
    set_error("univtg_adamw_step: buffers must be 16-byte aligned with n %% 4 == 0, step >= 1, scratch non-null");
    return (int)cudaErrorInvalidValue;
  }
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const size_t n4 = n / 4;
  size_t blocks = (n4 + 255) / 256;
  if (blocks > (size_t)sms * 8) blocks = (size_t)sms * 8;
  if (blocks > UNIVTG_ADAMW_SCRATCH_FLOATS - 4) blocks = UNIVTG_ADAMW_SCRATCH_FLOATS - 4;
  launch_k(sumsq_kernel, dim3((unsigned)blocks), dim3(256), 0, st, grads, n4, scratch2 + 4);
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
  a.bc1 = (float)(1.0 - pow((double)beta1, (double)step));
  a.bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
  a.max_norm = max_grad_norm;
  a.scratch = scratch2;
  a.n_partial = (int)blocks;
  a.g_out = write_clipped_grads ? grads : nullptr;
  if (segs != nullptr && segs->n > 0) {
    launch_k(adamw_kernel<true>, dim3((unsigned)blocks), dim3(256), 0, st, a, *segs);
  } else {
    PackSegTable none;
    none.n = 0;
    none.fmt = 0;
    launch_k(adamw_kernel<false>, dim3((unsigned)blocks), dim3(256), 0, st, a, none);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_adamw_step launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}
}  // namespace uv
