// CLIP-teacher pseudo labels (reference teacher/clip2label.py): for every video the top-k classes by the sum over its clips of
// the clip-class cosines, and for each of them the per-clip curve cos // th with the windows of its maximum.
//
//   univtg_teacher_prepare_classes  once per class table: fp64 norms, normalised rows as fp16 hi / lo planes (rows padded to
//                                   a multiple of 16, K to a multiple of 64).
//   univtg_teacher_label            per chunk of videos:
//     pool_kernel        one block per video: fp64 clip norms, the mean normalised clip row as fp16 hi / lo planes, its norm.
//     univtg_op_gemm     fmt 2 (fp16x3), ksplit 1: approximate mean cosines [V, C_pad] (sum over clips / T).
//     candidates_kernel  one block per video: the kR best approximate columns (ties to the lower index) and the (kR+1)-th value.
//     score_kernel       one block per video: exact fp64 sums of the candidates, the top-k by (sum desc, index asc), the
//                        certificate that no other class can reach the k-th, and the curves and windows of the chosen classes.
//                        Videos that fail the certificate are flagged, and a second launch of the same kernel rescores them
//                        over every class.
// Sums over clips run in clip order inside one warp, and a class's dot products do not depend on where the class sits in a
// list, so duplicated class rows get bit-identical sums and the tie rule alone orders them.
#include <cuda_fp16.h>
#include <math.h>
#include <stdint.h>

#include "../../include/univtg_b200.h"
#include "kernels.h"
#include "ptx.cuh"

// Python's float // (CPython Objects/floatobject.c, float_floor_div -> _float_div_mod): fmod, the remainder's sign fix-up, the
// quotient snapped to the nearest integer, and a zero quotient signed like the true quotient.  1.0 // 0.05 is 19.0, not
// floor(1.0 / 0.05) = 20.  Host and device run the same IEEE double operations (fmod, floor and copysign are exact).
#ifdef __CUDA_ARCH__
#define UV_DSUB(a, b) __dsub_rn(a, b)
#define UV_DADD(a, b) __dadd_rn(a, b)
#define UV_DDIV(a, b) __ddiv_rn(a, b)
#else
#define UV_DSUB(a, b) ((a) - (b))
#define UV_DADD(a, b) ((a) + (b))
#define UV_DDIV(a, b) ((a) / (b))
#endif
__host__ __device__ inline double py_floordiv(double vx, double wx) {
  double mod = fmod(vx, wx);
  double div = UV_DDIV(UV_DSUB(vx, mod), wx);
  if (mod != 0.0) {
    if ((wx < 0.0) != (mod < 0.0)) {
      mod = UV_DADD(mod, wx);
      div = UV_DSUB(div, 1.0);
    }
  }
  if (div != 0.0) {
    double fl = floor(div);
    if (UV_DSUB(div, fl) > 0.5) fl = UV_DADD(fl, 1.0);
    return fl;
  }
  return copysign(0.0, UV_DDIV(vx, wx));
}

namespace uv {
namespace {

constexpr int kR = 16;          // approximate candidates per video (>= topk)
constexpr int kMaxK = 16;       // topk
constexpr int kMaxD = 1024;     // feature width: a class row lives in 32 registers per lane
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kBinNegZero = INT32_MIN;  // a bin of -0.0

__host__ __device__ inline int pad16(int x) { return (x + 15) / 16 * 16; }
__host__ __device__ inline int pad64(int x) { return (x + 63) / 64 * 64; }
inline size_t al256(size_t x) { return (x + 255) / 256 * 256; }

// fp64 sum over the block in a fixed order (per thread, warp butterfly, then warp 0..7); every thread gets the result
__device__ double block_sum(double x, double* s_red) {
#pragma unroll
  for (int off = 16; off; off >>= 1) x = __dadd_rn(x, __shfl_xor_sync(0xffffffffu, x, off));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = x;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < kWarps; ++w) s = __dadd_rn(s, s_red[w]);
  return s;
}

__device__ __forceinline__ void split_store(double x, __half* hi, __half* lo) {
  const __half h = __double2half(x);
  *hi = h;
  *lo = __double2half(__dsub_rn(x, (double)__half2float(h)));
}

struct ClassWs {
  __half* planes;  // [2][C_pad][Dp]
  double* norm;    // [C_pad] max(||c||, 1e-8)
};
inline ClassWs class_ws(void* ws, int C, int D) {
  const size_t planes = al256((size_t)2 * pad16(C) * pad64(D) * sizeof(__half));
  char* p = static_cast<char*>(ws);
  return ClassWs{reinterpret_cast<__half*>(p), reinterpret_cast<double*>(p + planes)};
}
inline size_t class_ws_bytes(int C, int D) {
  return al256((size_t)2 * pad16(C) * pad64(D) * sizeof(__half)) + al256((size_t)pad16(C) * sizeof(double));
}

struct ChunkWs {
  double* clip_norm;  // [S]
  double* clip_inv;   // [S] 1 / clip_norm (the pooled row only feeds the approximate ranking)
  __half* planes;     // [2][V][Dp]
  double* mean_norm;  // [V]
  float* approx;      // [V][C_pad]
  int32_t* cand;      // [V][kR]
  float* next;        // [V] the (kR+1)-th approximate value
  int32_t* flag;      // [V] 1: rescore over every class
};
inline size_t chunk_ws_bytes(int V, long long S, int C, int D, ChunkWs* out, void* base) {
  size_t o = 0;
  char* p = static_cast<char*>(base);
  auto take = [&](size_t bytes) {
    char* r = p ? p + o : nullptr;
    o += al256(bytes);
    return r;
  };
  ChunkWs w;
  w.clip_norm = reinterpret_cast<double*>(take((size_t)S * sizeof(double)));
  w.clip_inv = reinterpret_cast<double*>(take((size_t)S * sizeof(double)));
  w.planes = reinterpret_cast<__half*>(take((size_t)2 * V * pad64(D) * sizeof(__half)));
  w.mean_norm = reinterpret_cast<double*>(take((size_t)V * sizeof(double)));
  w.approx = reinterpret_cast<float*>(take((size_t)V * pad16(C) * sizeof(float)));
  w.cand = reinterpret_cast<int32_t*>(take((size_t)V * kR * sizeof(int32_t)));
  w.next = reinterpret_cast<float*>(take((size_t)V * sizeof(float)));
  w.flag = reinterpret_cast<int32_t*>(take((size_t)V * sizeof(int32_t)));
  if (out) *out = w;
  return o;
}

// ---- class table ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) class_prep_kernel(const float* __restrict__ cls, int C, int D, ClassWs w) {
  pdl_prologue();
  __shared__ double s_red[kWarps];
  const int c = blockIdx.x, Cp = gridDim.x, Dp = pad64(D);
  const float* row = cls + (size_t)c * D;
  double ss = 0.0;
  if (c < C)
    for (int i = threadIdx.x; i < D; i += kThreads) ss = __fma_rn((double)row[i], (double)row[i], ss);
  const double n = fmax(__dsqrt_rn(block_sum(ss, s_red)), 1e-8);
  if (threadIdx.x == 0) w.norm[c] = n;
  for (int i = threadIdx.x; i < Dp; i += kThreads) {
    const double x = (c < C && i < D) ? __ddiv_rn((double)row[i], n) : 0.0;
    split_store(x, w.planes + (size_t)c * Dp + i, w.planes + (size_t)Cp * Dp + (size_t)c * Dp + i);
  }
}

// ---- per video: clip norms and the mean normalised row -------------------------------------------------------------------
struct PoolArgs {
  const float* feats;   // [S, D]
  const int32_t* off;   // [V + 1]
  int V, D;
  ChunkWs w;
};

__global__ void __launch_bounds__(kThreads) pool_kernel(const PoolArgs a) {
  pdl_prologue();
  __shared__ double s_red[kWarps];
  const int v = blockIdx.x, lane = threadIdx.x & 31, wp = threadIdx.x >> 5, D = a.D, Dp = pad64(D);
  const int off = a.off[v], T = a.off[v + 1] - off;
  const float* x = a.feats + (size_t)off * D;
  for (int t = wp; t < T; t += kWarps) {
    double ss = 0.0;
    for (int i = lane; i < D; i += 32) ss = __fma_rn((double)x[(size_t)t * D + i], (double)x[(size_t)t * D + i], ss);
#pragma unroll
    for (int o = 16; o; o >>= 1) ss = __dadd_rn(ss, __shfl_xor_sync(0xffffffffu, ss, o));
    const double n = fmax(__dsqrt_rn(ss), 1e-8);
    if (lane == 0) {
      a.w.clip_norm[off + t] = n;
      a.w.clip_inv[off + t] = __drcp_rn(n);
    }
  }
  __syncthreads();
  const double* inv = a.w.clip_inv + off;
  double sq = 0.0;
  for (int i = threadIdx.x; i < Dp; i += kThreads) {
    double m = 0.0;
    if (i < D) {
      for (int t = 0; t < T; ++t) m = __fma_rn((double)x[(size_t)t * D + i], inv[t], m);
      m = __dmul_rn(m, __drcp_rn((double)T));
    }
    sq = __fma_rn(m, m, sq);
    split_store(m, a.w.planes + (size_t)v * Dp + i, a.w.planes + (size_t)a.V * Dp + (size_t)v * Dp + i);
  }
  const double n = __dsqrt_rn(block_sum(sq, s_red));
  if (threadIdx.x == 0) a.w.mean_norm[v] = n;
}

// ---- approximate candidates -----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t order_key(float x) {  // unsigned key with the order of x (finite values; -0 == +0)
  uint32_t u = __float_as_uint(x);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// keys (value, ~index): the largest key is the largest value, then the lowest index; 0 = no column
__global__ void __launch_bounds__(kThreads) candidates_kernel(const float* __restrict__ approx, int C, int Cp, int32_t* cand,
                                                              float* next) {
  pdl_prologue();
  __shared__ unsigned long long s_red[kWarps];
  const int v = blockIdx.x;
  const float* row = approx + (size_t)v * Cp;
  unsigned long long prev = ~0ull;
  for (int r = 0; r <= kR; ++r) {
    unsigned long long best = 0ull;
    for (int c = threadIdx.x; c < C; c += kThreads) {
      const unsigned long long k = ((unsigned long long)order_key(row[c]) << 32) | (0xffffffffu - (uint32_t)c);
      if (k < prev && k > best) best = k;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o);
      best = ob > best ? ob : best;
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = best;
    __syncthreads();
    best = 0ull;
    for (int w = 0; w < kWarps; ++w) best = s_red[w] > best ? s_red[w] : best;
    if (threadIdx.x == 0) {
      if (r < kR) cand[v * kR + r] = best ? (int32_t)(0xffffffffu - (uint32_t)best) : -1;
      else next[v] = best ? key_value((uint32_t)(best >> 32)) : -INFINITY;
    }
    prev = best;
    if (!best) {
      for (int q = r + 1 + threadIdx.x; q <= kR; q += kThreads) {
        if (q < kR) cand[v * kR + q] = -1;
        else next[v] = -INFINITY;
      }
      break;
    }
  }
}

// ---- exact sums, top-k, certificate, curves -------------------------------------------------------------------------------
struct ScoreArgs {
  const float* feats;     // [S, D]
  const int32_t* off;     // [V + 1]
  const float* cls;       // [C, D]
  const double* cls_norm; // [C]
  int V, C, D, K, all;    // all = 1: the fallback pass over every class, for flagged videos only
  double th, e_rel, e_abs;
  ChunkWs w;
  int32_t* idx;    // [V, K]
  int32_t* nwin;   // [V, K]
  uint32_t* win;   // [S, K] (first clip << 16) | last clip of each window
  int32_t* bins;   // [S, K]
  int32_t* count;  // fallback videos
};

__device__ __forceinline__ bool better(double sa, int ia, double sb, int ib) { return sa > sb || (sa == sb && ia < ib); }

__device__ __forceinline__ void load_row(const float* row, int D, int lane, float (&r)[kMaxD / 32]) {
#pragma unroll
  for (int k = 0; k < kMaxD / 32; ++k) {
    const int i = lane + 32 * k;
    r[k] = (row && i < D) ? row[i] : 0.0f;
  }
}

// fp64 dot of clip row x with the register row r, in a fixed order; every lane returns the same value
__device__ __forceinline__ double warp_dot(const float* x, int D, int lane, const float (&r)[kMaxD / 32]) {
  double d = 0.0;
#pragma unroll
  for (int k = 0; k < kMaxD / 32; ++k) {
    const int i = lane + 32 * k;
    if (i < D) d = __fma_rn((double)x[i], (double)r[k], d);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) d = __dadd_rn(d, __shfl_xor_sync(0xffffffffu, d, o));
  return d;
}

__global__ void __launch_bounds__(kThreads) score_kernel(const ScoreArgs a) {
  pdl_prologue();
  __shared__ double s_ls[kWarps][kMaxK];
  __shared__ int s_li[kWarps][kMaxK];
  __shared__ int s_ln[kWarps];
  __shared__ double s_top[kMaxK];
  __shared__ int s_topi[kMaxK];
  __shared__ int s_k;
  const int v = blockIdx.x, lane = threadIdx.x & 31, wp = threadIdx.x >> 5, D = a.D, K = a.K;
  if (a.all && !a.w.flag[v]) return;
  const int off = a.off[v], T = a.off[v + 1] - off;
  const float* x = a.feats + (size_t)off * D;
  const double* nv = a.w.clip_norm + off;
  if (lane == 0) s_ln[wp] = 0;

  // exact sums of candidate pairs; lane 0 keeps the warp's best K
  const int npairs = a.all ? (a.C + 1) / 2 : kR / 2;
  for (int p = wp; p < npairs; p += kWarps) {
    int c0, c1;
    if (a.all) {
      c0 = 2 * p;
      c1 = 2 * p + 1 < a.C ? 2 * p + 1 : -1;
    } else {
      c0 = a.w.cand[v * kR + 2 * p];
      c1 = a.w.cand[v * kR + 2 * p + 1];
    }
    if (c0 < 0) continue;
    float r0[kMaxD / 32], r1[kMaxD / 32];
    load_row(a.cls + (size_t)c0 * D, D, lane, r0);
    load_row(c1 >= 0 ? a.cls + (size_t)c1 * D : nullptr, D, lane, r1);
    const double n0 = a.cls_norm[c0], n1 = c1 >= 0 ? a.cls_norm[c1] : 1.0;
    double s0 = 0.0, s1 = 0.0;
    for (int t = 0; t < T; ++t) {
      const float* xt = x + (size_t)t * D;
      s0 = __dadd_rn(s0, __ddiv_rn(warp_dot(xt, D, lane, r0), __dmul_rn(nv[t], n0)));
      if (c1 >= 0) s1 = __dadd_rn(s1, __ddiv_rn(warp_dot(xt, D, lane, r1), __dmul_rn(nv[t], n1)));
    }
    if (lane == 0) {
      for (int q = 0; q < 2; ++q) {
        const int c = q ? c1 : c0;
        const double s = q ? s1 : s0;
        if (c < 0) continue;
        int n = s_ln[wp], j = n < K ? n : K;
        if (n == K && !better(s, c, s_ls[wp][K - 1], s_li[wp][K - 1])) continue;
        if (j == K) --j;  // drop the last
        while (j > 0 && better(s, c, s_ls[wp][j - 1], s_li[wp][j - 1])) {
          s_ls[wp][j] = s_ls[wp][j - 1];
          s_li[wp][j] = s_li[wp][j - 1];
          --j;
        }
        s_ls[wp][j] = s;
        s_li[wp][j] = c;
        if (n < K) s_ln[wp] = n + 1;
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // merge the warps' lists
    int head[kWarps];
    for (int w = 0; w < kWarps; ++w) head[w] = 0;
    int k = 0;
    for (; k < K; ++k) {
      int bw = -1;
      for (int w = 0; w < kWarps; ++w)
        if (head[w] < s_ln[w] && (bw < 0 || better(s_ls[w][head[w]], s_li[w][head[w]], s_ls[bw][head[bw]], s_li[bw][head[bw]])))
          bw = w;
      if (bw < 0) break;
      s_top[k] = s_ls[bw][head[bw]];
      s_topi[k] = s_li[bw][head[bw]];
      ++head[bw];
    }
    // certificate: every other class c has approx_c <= next and |approx_c - exact_c / T| <= e, so it stays below the k-th
    // exact sum when that exceeds T * (next + 2 e)
    bool ok = true;
    if (!a.all && k == K) {
      const double nxt = (double)a.w.next[v];
      if (nxt != -INFINITY) {
        const double e = __fma_rn(a.e_rel, a.w.mean_norm[v], a.e_abs);
        ok = s_top[K - 1] > __dmul_rn((double)T, __fma_rn(2.0, e, nxt));
      }
    }
    if (!ok) {
      a.w.flag[v] = 1;
      atomicAdd(a.count, 1);
      k = -1;
    }
    s_k = k;
  }
  __syncthreads();
  const int k = s_k;
  if (k < 0) return;

  // curves: float32(cos) // th per clip, and the runs of the maximum that end before the last clip
  for (int r = wp; r < K; r += kWarps) {
    int32_t* b = a.bins + (size_t)off * K + r;
    if (r >= k) {
      if (lane == 0) {
        a.idx[v * K + r] = -1;
        a.nwin[v * K + r] = 0;
      }
      continue;
    }
    const int c = s_topi[r];
    float cr[kMaxD / 32];
    load_row(a.cls + (size_t)c * D, D, lane, cr);
    const double nc = a.cls_norm[c];
    double mx = -INFINITY;
    for (int t = 0; t < T; ++t) {
      const double cs = __ddiv_rn(warp_dot(x + (size_t)t * D, D, lane, cr), __dmul_rn(nv[t], nc));
      const double q = py_floordiv((double)__double2float_rn(cs), a.th);
      mx = fmax(mx, q);
      if (lane == 0) b[(size_t)t * K] = (q == 0.0 && signbit(q)) ? kBinNegZero : (int32_t)q;
    }
    if (lane == 0) {
      const int32_t m = (int32_t)mx;
      int n = 0, start = -1;
      for (int t = 0; t < T; ++t) {
        const int32_t q = b[(size_t)t * K];
        const bool at_max = (q == kBinNegZero ? 0 : q) == m;
        if (at_max && start < 0) start = t;
        if (!at_max && start >= 0) {
          a.win[(size_t)(off + n) * K + r] = ((uint32_t)start << 16) | (uint32_t)(t - 1);
          ++n;
          start = -1;
        }
      }
      a.idx[v * K + r] = c;
      a.nwin[v * K + r] = n;
    }
  }
}

}  // namespace
}  // namespace uv

extern "C" size_t univtg_teacher_class_bytes(int32_t C, int32_t D) {
  if (C < 1 || D < 1 || D > uv::kMaxD) {
    uv::set_error("univtg_teacher_class_bytes: C must be >= 1 and D in 1..%d", uv::kMaxD);
    return 0;
  }
  return uv::class_ws_bytes(C, D);
}

extern "C" int univtg_teacher_prepare_classes(const float* cls, int32_t C, int32_t D, void* ws, void* stream) {
  using namespace uv;
  if (!cls || !ws || C < 1 || D < 1 || D > kMaxD) {
    set_error("univtg_teacher_prepare_classes: bad argument (C >= 1, D in 1..%d)", kMaxD);
    return 1;
  }
  launch_k(class_prep_kernel, dim3(pad16(C)), dim3(kThreads), 0, reinterpret_cast<cudaStream_t>(stream), cls, (int)C, (int)D,
           class_ws(ws, C, D));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_teacher_prepare_classes launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

extern "C" size_t univtg_teacher_chunk_bytes(int32_t V, int64_t S, int32_t C, int32_t D) {
  if (V < 1 || S < V || C < 1 || D < 1 || D > uv::kMaxD) {
    uv::set_error("univtg_teacher_chunk_bytes: bad argument (V >= 1, S >= V, C >= 1, D in 1..%d)", uv::kMaxD);
    return 0;
  }
  return uv::chunk_ws_bytes(V, S, C, D, nullptr, nullptr);
}

extern "C" int univtg_teacher_label(const float* cls, const void* cls_ws, int32_t C, int32_t D, const float* feats,
                                    const int32_t* offsets, int32_t V, int64_t S, int32_t topk, double th, void* ws,
                                    size_t ws_bytes, int32_t* out, void* stream) {
  using namespace uv;
  if (!cls || !cls_ws || !feats || !offsets || !ws || !out || C < 1 || D < 1 || D > kMaxD || V < 1 || S < V || topk < 1 ||
      topk > kMaxK || !(th >= 0x1p-30) || !isfinite(th)) {
    set_error("univtg_teacher_label: bad argument (C >= 1, D in 1..%d, V >= 1, S >= V, topk in 1..%d, finite th >= 2^-30)",
              kMaxD, kMaxK);
    return 1;
  }
  ChunkWs w;
  if (chunk_ws_bytes(V, S, C, D, &w, ws) > ws_bytes) {
    set_error("univtg_teacher_label: workspace too small (univtg_teacher_chunk_bytes)");
    return 1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int K = topk, Cp = pad16(C), Dp = pad64(D);
  const ClassWs cw = class_ws(const_cast<void*>(cls_ws), C, D);
  int32_t* idx = out;
  int32_t* nwin = idx + (size_t)V * K;
  uint32_t* win = reinterpret_cast<uint32_t*>(nwin + (size_t)V * K);
  int32_t* bins = reinterpret_cast<int32_t*>(win + (size_t)S * K);
  int32_t* count = bins + (size_t)S * K;
  cudaError_t e = cudaMemsetAsync(out, 0, ((size_t)2 * V * K + (size_t)2 * S * K + 1) * sizeof(int32_t), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(w.flag, 0, (size_t)V * sizeof(int32_t), st);
  if (e != cudaSuccess) {
    set_error("univtg_teacher_label: %s", cudaGetErrorString(e));
    return (int)e;
  }
  launch_k(pool_kernel, dim3(V), dim3(kThreads), 0, st, PoolArgs{feats, offsets, (int)V, (int)D, w});
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int32_t Ms[1] = {V}, Ns[1] = {Cp}, kb[1] = {Dp / 64};
  const TileChoice tc = choose_tile(Ms, Ns, kb, 1, sms, 16, 1);
  int rc = univtg_op_gemm(w.planes, cw.planes, V, Cp, Dp, 0, 0, 2, tc.bn, 1, nullptr, 0, 1.0f, w.approx, nullptr, stream);
  if (rc) return rc;
  launch_k(candidates_kernel, dim3(V), dim3(kThreads), 0, st, (const float*)w.approx, (int)C, Cp, w.cand, w.next);
  // |approx - exact / T| for a class of norm <= 1 and a mean row of norm n: the dropped lo x lo products and the residuals of
  // the two splits add at most 3 * 2^-22 n plus 2^-25 per element for fp16 subnormals (<= 2^-25 sqrt(D) in total, per side);
  // the fp32 accumulation of 3D exact products adds at most 3D * 2^-23 * (1 + 2^-10) n, rounding by truncation included.
  // e_rel and e_abs round both up (a deliberately generous bound).
  const double e_rel = 3.0 * D * 0x1p-23 + 0x1p-19, e_abs = 0x1p-23 * sqrt((double)D);
  ScoreArgs sa{feats, offsets, cls, cw.norm, (int)V, (int)C, (int)D, K, 0, th, e_rel, e_abs, w, idx, nwin, win, bins, count};
  launch_k(score_kernel, dim3(V), dim3(kThreads), 0, st, sa);
  sa.all = 1;
  launch_k(score_kernel, dim3(V), dim3(kThreads), 0, st, sa);
  e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_teacher_label launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

extern "C" int univtg_debug_py_floordiv(const double* x, int64_t n, double th, double* out) {
  if ((!x || !out) && n > 0) {
    uv::set_error("univtg_debug_py_floordiv: null argument");
    return 1;
  }
  if (n < 0 || th == 0.0) {
    uv::set_error("univtg_debug_py_floordiv: n must be >= 0 and th nonzero");
    return 1;
  }
  for (int64_t i = 0; i < n; ++i) out[i] = py_floordiv(x[i], th);
  return 0;
}
