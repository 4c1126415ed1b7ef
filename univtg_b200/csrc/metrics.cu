// Per-query metrics of the reference's eval_submission (eval/eval.py, eval/utils.py), on the device.
//   univtg_eval_mr  compute_average_precision_detection (AP at IoU 0.50:0.05:0.95 over the first 10 windows), the R1 and R5 IoUs,
//                   for the length ranges (0,10], (10,30], (30,inf) and the full set: one block per query, one warp per range.
//   univtg_eval_hl  get_ap over scikit-learn's precision_recall_curve and HIT@1 for min scores 2/3/4 x 3 annotators: one block
//                   per query, one sort of the predicted scores shared by the 9 curves, one warp per curve.
// Everything is IEEE double with explicit _rn intrinsics (no FMA contraction), so every per-query value equals numpy's bit for
// bit; the short sums inside a query follow numpy's pairwise summation (pairwise_sum below).  The means over queries stay on the
// host, in numpy.
#include <math.h>
#include <stdint.h>

#include "../../include/univtg_b200.h"
#include "kernels.h"
#include "ptx.cuh"

namespace uv {
namespace {

constexpr int kMaxPred = 10;    // windows per query the metrics read: AP the first 10, R5 the first 5, R1 the first one
constexpr int kMaxGt = 64;      // gt windows per query (one 64-bit lock mask per threshold)
constexpr int kMaxClips = 4096; // int(duration / 2) per query (the decode bound)
constexpr int kThds = 10;
constexpr int kHlThreads = 288;  // 9 warps: min score 2/3/4 x annotator
// float(f"{e:.2f}") for e in np.linspace(0.5, 0.95, 10): the doubles nearest to these decimals, as the literals below are
__constant__ double kIouThd[kThds] = {0.5, 0.55, 0.6, 0.65, 0.7, 0.75, 0.8, 0.85, 0.9, 0.95};

// numpy's sum of a contiguous float64 vector (np.add.reduce -> pairwise_sum): below 8 elements a plain loop from -0.0; up to
// 128 eight interleaved accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the remainder in order; above 128
// the halves [0, n2) and [n2, n) with n2 = n/2 rounded down to a multiple of 8.  a[i * stride] is element i.
__device__ __noinline__ double pairwise_leaf(const double* a, int n, int stride) {
  if (n < 8) {
    double r = -0.0;
    for (int i = 0; i < n; ++i) r = __dadd_rn(r, a[i * stride]);
    return r;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = a[j * stride];
  int i = 8;
  for (; i < n - (n % 8); i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[(i + j) * stride]);
  }
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __dadd_rn(res, a[i * stride]);
  return res;
}

template <int kDepth>  // n <= 128 * 2^kDepth
__device__ double pairwise_sum(const double* a, int n, int stride) {
  if constexpr (kDepth == 0) {
    return pairwise_leaf(a, n, stride);
  } else {
    if (n <= 128) return pairwise_leaf(a, n, stride);
    int n2 = n / 2;
    n2 -= n2 % 8;
    return __dadd_rn(pairwise_sum<kDepth - 1>(a, n2, stride), pairwise_sum<kDepth - 1>(a + (ptrdiff_t)n2 * stride, n - n2, stride));
  }
}

// compute_temporal_iou_batch_cross for one pair: inter / ((len p + len g) - inter); 0/0 gives NaN as in numpy
__device__ __forceinline__ double cross_iou(double ps, double pe, double gs, double ge) {
  const double x = __dsub_rn(fmin(pe, ge), fmax(ps, gs));
  const double inter = x > 0.0 ? x : 0.0;
  return __ddiv_rn(inter, __dsub_rn(__dadd_rn(__dsub_rn(pe, ps), __dsub_rn(ge, gs)), inter));
}

// compute_temporal_iou_batch_paired: intersection over the convex hull, 0 where the hull is empty
__device__ __forceinline__ double paired_iou(double ps, double pe, double gs, double ge) {
  const double inter = fmax(0.0, __dsub_rn(fmin(pe, ge), fmax(ps, gs)));
  const double hull = __dsub_rn(fmax(pe, ge), fmin(ps, gs));
  return hull != 0.0 ? __ddiv_rn(inter, hull) : 0.0;
}

struct MrArgs {
  const double* pred;     // [Q, 10, 3] st, ed, score in submission order
  const int32_t* n_pred;  // [Q] in 1..10
  const double* gt;       // [Q, G, 2]
  const int32_t* n_gt;    // [Q] in 1..G
  double* ap;             // [4, Q, 10]
  double* iou_r1;         // [4, Q]
  double* iou_r5;         // [4, Q]
  uint8_t* kept;          // [4, Q]
  int Q, G;
};

__global__ void __launch_bounds__(128) eval_mr_kernel(const MrArgs a) {
  pdl_prologue();
  __shared__ double s_p[kMaxPred][3];
  __shared__ double s_g[kMaxGt][2];
  __shared__ int s_ord[kMaxPred];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, r = tid >> 5;
  const int np = a.n_pred[q], ng = a.n_gt[q];
  for (int i = tid; i < np * 3; i += blockDim.x) s_p[i / 3][i % 3] = a.pred[(size_t)q * kMaxPred * 3 + i];
  for (int i = tid; i < ng * 2; i += blockDim.x) s_g[i / 2][i % 2] = a.gt[(size_t)q * a.G * 2 + i];
  __syncthreads();
  if (tid == 0) {  // prediction.sort(key=-score): stable insertion sort
    for (int k = 0; k < np; ++k) {
      int j = k;
      while (j > 0 && s_p[s_ord[j - 1]][2] < s_p[k][2]) {
        s_ord[j] = s_ord[j - 1];
        --j;
      }
      s_ord[j] = k;
    }
  }
  __syncthreads();
  // get_data_by_range: the gt windows with lo < ed - st <= hi (every window for the full set)
  const double lo = r == 1 ? 10.0 : r == 2 ? 30.0 : 0.0, hi = r == 0 ? 10.0 : r == 1 ? 30.0 : INFINITY;
  uint64_t in = 0;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int j = h * 32 + lane;
    bool b = false;
    if (j < ng) {
      const double len = __dsub_rn(s_g[j][1], s_g[j][0]);
      b = r == 3 || (lo < len && len <= hi);
    }
    in |= (uint64_t)__ballot_sync(0xffffffffu, b) << (32 * h);
  }
  const int M = __popcll(in);
  const size_t o = (size_t)r * a.Q + q;
  if (M == 0) {  // this query is not in the range
    if (lane < kThds) a.ap[o * kThds + lane] = 0.0;
    if (lane == 0) {
      a.kept[o] = 0;
      a.iou_r1[o] = 0.0;
      a.iou_r5[o] = 0.0;
    }
    return;
  }
  if (lane < kThds) {
    // Greedy matching at one threshold.  The reference visits the gt windows in argsort()[::-1] order (NaN first, then
    // decreasing IoU, ties to the higher index), skips locked ones and stops at the first IoU below the threshold: the
    // prediction is a true positive exactly when the first unlocked window in that order does not have IoU < thd.
    const double thd = kIouThd[lane];
    uint64_t lock = 0;
    double mp[kMaxPred + 2], mr[kMaxPred + 2], terms[kMaxPred + 1];
    mp[0] = 0.0;
    mr[0] = 0.0;
    int tp = 0;
    for (int k = 0; k < np; ++k) {
      const int p = s_ord[k];
      int best = -1;
      double bv = 0.0;
      for (uint64_t m = in & ~lock; m; m &= m - 1) {
        const int j = __ffsll((long long)m) - 1;
        const double v = cross_iou(s_p[p][0], s_p[p][1], s_g[j][0], s_g[j][1]);
        if (best < 0 || isnan(v) || (!isnan(bv) && v >= bv)) {
          best = j;
          bv = v;
        }
      }
      if (best >= 0 && !(bv < thd)) {
        lock |= 1ull << best;
        ++tp;
      }
      mp[k + 1] = __ddiv_rn((double)tp, (double)(k + 1));  // tp / (tp + fp)
      mr[k + 1] = __ddiv_rn((double)tp, (double)M);
    }
    // interpolated_precision_recall
    mp[np + 1] = 0.0;
    mr[np + 1] = 1.0;
    double run = 0.0;  // running maximum from the end, carried in a register
    for (int i = np; i >= 0; --i) {
      if (mp[i] > run) run = mp[i];
      mp[i] = run;
    }
    int nt = 0;
    for (int i = 1; i <= np + 1; ++i)
      if (mr[i] != mr[i - 1]) terms[nt++] = __dmul_rn(__dsub_rn(mr[i], mr[i - 1]), mp[i]);
    a.ap[o * kThds + lane] = pairwise_leaf(terms, nt, 1);
  } else if (lane == kThds) {
    // R1: the first window against the gt window of highest IoU (np.argmax: the first maximum, a NaN wins)
    int best = -1;
    double bv = 0.0;
    for (uint64_t m = in; m; m &= m - 1) {
      const int j = __ffsll((long long)m) - 1;
      const double v = cross_iou(s_p[0][0], s_p[0][1], s_g[j][0], s_g[j][1]);
      if (best < 0 || (!isnan(bv) && (isnan(v) || v > bv))) {
        best = j;
        bv = v;
      }
    }
    a.iou_r1[o] = paired_iou(s_p[0][0], s_p[0][1], s_g[best][0], s_g[best][1]);
    a.kept[o] = 1;
  } else if (lane == kThds + 1) {
    // R5: IoUs of the first 5 windows x gt windows with NaN -> 0; the first maximum in row-major order
    int bp = -1, bg = -1;
    double bv = 0.0;
    const int n5 = np < 5 ? np : 5;
    for (int p = 0; p < n5; ++p) {
      for (uint64_t m = in; m; m &= m - 1) {
        const int j = __ffsll((long long)m) - 1;
        double v = cross_iou(s_p[p][0], s_p[p][1], s_g[j][0], s_g[j][1]);
        if (isnan(v)) v = 0.0;
        if (bp < 0 || v > bv) {
          bp = p;
          bg = j;
          bv = v;
        }
      }
    }
    a.iou_r5[o] = paired_iou(s_p[bp][0], s_p[bp][1], s_g[bg][0], s_g[bg][1]);
  }
}

struct HlArgs {
  const double* sal;       // [Q, S] predicted saliency, zero padded
  const int32_t* n_sal;    // [Q] >= 1
  const uint16_t* labels;  // [Q, C] bit (3 * level + annotator) = (gt score >= 2 + level)
  const int32_t* n_clips;  // [Q] int(duration / 2), 1..C
  double* scratch;         // [Q, 9, C]
  double* ap;              // [3, Q, 3]
  double* hit;             // [3, Q, 3]
  int Q, S, C, npad;
};

// sorted position a precedes b: larger score first, ties in clip order; padding (index >= n) last
__device__ __forceinline__ bool hl_precedes(double sa, int ia, double sb, int ib, int n) {
  if (ia >= n || ib >= n) return ia < ib;
  return sa > sb || (sa == sb && ia < ib);
}

// argmax order: a NaN beats everything, then the larger value, then the smaller index
__device__ __forceinline__ bool argmax_better(double va, int ia, double vb, int ib) {
  if (ib < 0) return ia >= 0;
  if (ia < 0) return false;
  if (isnan(va) != isnan(vb)) return isnan(va);
  if (!isnan(va) && va != vb) return va > vb;
  return ia < ib;
}

__global__ void __launch_bounds__(kHlThreads) eval_hl_kernel(const HlArgs a) {
  pdl_prologue();
  extern __shared__ uint8_t sm_raw[];
  double* s_key = reinterpret_cast<double*>(sm_raw);     // [npad]
  int* s_idx = reinterpret_cast<int*>(s_key + a.npad);   // [npad]
  uint16_t* s_lab = reinterpret_cast<uint16_t*>(s_idx + a.npad);  // [npad] labels in sorted order
  __shared__ double s_bv[kHlThreads / 32];
  __shared__ int s_bi[kHlThreads / 32];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5, nt = blockDim.x;
  const int n = a.n_clips[q], ns = a.n_sal[q];
  const double* sal = a.sal + (size_t)q * a.S;
  const uint16_t* lab = a.labels + (size_t)q * a.C;

  // HIT@1: np.argmax over the whole predicted list
  double bv = 0.0;
  int bi = -1;
  for (int i = tid; i < ns; i += nt) {
    const double v = sal[i];
    if (argmax_better(v, i, bv, bi)) {
      bv = v;
      bi = i;
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (argmax_better(ov, oi, bv, bi)) {
      bv = ov;
      bi = oi;
    }
  }
  if (lane == 0) {
    s_bv[w] = bv;
    s_bi[w] = bi;
  }
  // compute_ap_from_tuple: the prediction cut or zero-padded to n clips
  for (int i = tid; i < a.npad; i += nt) {
    s_key[i] = i < n ? (i < ns ? sal[i] : 0.0) : 0.0;
    s_idx[i] = i;
  }
  __syncthreads();
  if (tid < 9) {
    bv = s_bv[0];
    bi = s_bi[0];
    for (int k = 1; k < kHlThreads / 32; ++k)
      if (argmax_better(s_bv[k], s_bi[k], bv, bi)) {
        bv = s_bv[k];
        bi = s_bi[k];
      }
    const int lv = tid / 3, an = tid % 3;
    a.hit[((size_t)lv * a.Q + q) * 3 + an] = bi < n ? (double)((lab[bi] >> tid) & 1) : 0.0;
  }
  // bitonic sort, descending score (the order precision_recall_curve walks its thresholds in)
  for (int k = 2; k <= a.npad; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < a.npad; i += nt) {
        const int p = i ^ j;
        if (p > i) {
          const bool up = (i & k) == 0;
          const double si = s_key[i], sp = s_key[p];
          const int ii = s_idx[i], ip = s_idx[p];
          if (up ? hl_precedes(sp, ip, si, ii, n) : hl_precedes(si, ii, sp, ip, n)) {
            s_key[i] = sp;
            s_key[p] = si;
            s_idx[i] = ip;
            s_idx[p] = ii;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < n; i += nt) s_lab[i] = lab[s_idx[i]];
  __syncthreads();

  // Warp w: the curve of label bit w.  The distinct thresholds end at sorted positions e (key[e] != key[e + 1]) with
  // tps = positives in [0, e] and precision tps / (e + 1).  get_ap reverses the curve, takes the running maximum of the
  // precision from the low-threshold end, and averages it at every point where the recall changes: the point of each
  // threshold group that contains a positive (recall is tps / P, and distinct tps stay distinct in float32 for P <= 4096).
  // So the values averaged are, for those groups in decreasing position, the maximum precision over positions >= e.
  double* buf = a.scratch + ((size_t)q * 9 + w) * a.C;
  int carry_cnt = 0, carry_end = 0;
  for (int base = 0; base < n; base += 32) {  // ascending: prefix counts; buf[e] = precision (sign bit set: no positive)
    const int i = base + lane;
    const bool valid = i < n;
    const int pos = valid ? (s_lab[i] >> w) & 1 : 0;
    const bool end = valid && (i == n - 1 || s_key[i] != s_key[i + 1]);
    int cnt = pos;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, cnt, off);
      if (lane >= off) cnt += v;
    }
    cnt += carry_cnt;
    const int e = end ? cnt : -1;
    int prev = e;  // exclusive max-scan of e: tps at the previous group end
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, prev, off);
      if (lane >= off) prev = max(prev, v);
    }
    int prev_ex = __shfl_up_sync(0xffffffffu, prev, 1);
    if (lane == 0) prev_ex = -1;
    prev_ex = max(prev_ex, carry_end);
    if (valid) {
      const double prec = end ? __ddiv_rn((double)cnt, (double)(i + 1)) : 0.0;
      buf[i] = (end && cnt > prev_ex) ? prec : -prec;
    }
    carry_cnt = __shfl_sync(0xffffffffu, cnt, 31);
    carry_end = max(carry_end, __shfl_sync(0xffffffffu, prev, 31));
  }
  const int npos = carry_cnt;
  __syncwarp();
  int count = 0;
  double m_carry = 0.0;
  for (int top = n - 1; top >= 0; top -= 32) {  // descending: running max, compaction into buf[n - 1 - rank]
    const int i = top - lane;
    const bool valid = i >= 0;
    const double v = valid ? buf[i] : -0.0;
    const bool sel = valid && !signbit(v);
    double m = fabs(v);
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const double u = __shfl_up_sync(0xffffffffu, m, off);
      if (lane >= off && u > m) m = u;
    }
    if (m_carry > m) m = m_carry;
    const unsigned ball = __ballot_sync(0xffffffffu, sel);
    const int rank = count + __popc(ball & ((1u << lane) - 1u));
    __syncwarp();
    if (sel) buf[n - 1 - rank] = m;
    m_carry = __shfl_sync(0xffffffffu, m, 31);
    count += __popc(ball);
  }
  __syncwarp();
  if (lane == 0) {
    const int lv = w / 3, an = w % 3;
    double ap;
    if (npos == 0) {
      ap = 0.0;  // every label 0
    } else if (npos == n) {
      ap = 1.0;  // every label 1
    } else {
      ap = __ddiv_rn(pairwise_sum<6>(buf + (n - 1), count, -1), (double)count);  // np.mean
    }
    a.ap[((size_t)lv * a.Q + q) * 3 + an] = ap;
  }
}

}  // namespace
}  // namespace uv

extern "C" int univtg_eval_mr(const double* pred, const int32_t* n_pred, const double* gt, const int32_t* n_gt, int32_t Q, int32_t G,
                              double* ap, double* iou_r1, double* iou_r5, uint8_t* kept, void* stream) {
  using namespace uv;
  if (!pred || !n_pred || !gt || !n_gt || !ap || !iou_r1 || !iou_r5 || !kept || Q < 0 || G < 1 || G > kMaxGt) {
    set_error("univtg_eval_mr: bad argument (G must be in 1..%d)", kMaxGt);
    return 1;
  }
  if (Q == 0) return 0;
  MrArgs a{pred, n_pred, gt, n_gt, ap, iou_r1, iou_r5, kept, Q, G};
  launch_k(eval_mr_kernel, dim3(Q), dim3(128), 0, reinterpret_cast<cudaStream_t>(stream), a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_eval_mr launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

extern "C" int univtg_eval_hl(const double* sal, const int32_t* n_sal, const uint16_t* labels, const int32_t* n_clips, int32_t Q,
                              int32_t S, int32_t C, double* scratch, double* ap, double* hit, void* stream) {
  using namespace uv;
  if (!sal || !n_sal || !labels || !n_clips || !scratch || !ap || !hit || Q < 0 || S < 1 || C < 1 || C > kMaxClips) {
    set_error("univtg_eval_hl: bad argument (C must be in 1..%d)", kMaxClips);
    return 1;
  }
  if (Q == 0) return 0;
  int npad = 1;
  while (npad < C) npad <<= 1;
  const size_t smem = (size_t)npad * (sizeof(double) + sizeof(int) + sizeof(uint16_t));
  cudaError_t e = cudaFuncSetAttribute(eval_hl_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    set_error("cudaFuncSetAttribute(eval_hl): %s", cudaGetErrorString(e));
    return (int)e;
  }
  HlArgs a{sal, n_sal, labels, n_clips, scratch, ap, hit, Q, S, C, npad};
  launch_k(eval_hl_kernel, dim3(Q), dim3(kHlThreads), smem, reinterpret_cast<cudaStream_t>(stream), a);
  e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_eval_hl launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}
