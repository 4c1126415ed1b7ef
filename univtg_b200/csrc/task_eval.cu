// Evaluation of the highlight-detection and video-summarisation task families, on the device.
//   univtg_eval_hl_topk  main/dataset.py DatasetHL.evaluate: one AP per (video, annotator) over the top of the score ranking
//                        (TVSum: label > lower median, the first k; YouTube: match > 0, the whole list).  One block per video.
//   univtg_qfvs_match    eval/qfvs.py calculate_semantic_matching: the total weight of a maximum-weight bipartite matching
//                        between machine-summary and ground-truth shots, weights the semantic IoU of their tag sets.  One block
//                        per query.
//   univtg_qfvs_eval_select  main/inference_qfvs.py eval_epoch: each query's score, its top k and the tag masks of the chosen
//                        shots, written into the epoch's pools.  One block per query.
// All arithmetic is IEEE double with explicit _rn intrinsics (no FMA contraction), so univtg_eval_hl_topk's APs equal the
// reference's Python floats bit for bit.
#include <math.h>
#include <stdint.h>

#include "../../include/univtg_b200.h"
#include "kernels.h"
#include "ptx.cuh"

namespace uv {
namespace {

constexpr int kMaxClips = 4096;   // clips per video (score row and label rows)
constexpr int kMaxAnno = 32;      // annotators: one warp each
constexpr int kMaxSide = 1024;    // shots on either side of a matching
constexpr int kMatchThreads = 256;
constexpr int kColsPerThread = kMaxSide / kMatchThreads;

// ---- torch.argsort(x, descending=True) on the CPU ----------------------------------------------------------------------
// ATen's CPU sort without stable=True is libstdc++'s std::sort over (value, index) pairs with the comparator "a > b" (NaN
// first; the host rejects non-finite scores).  std::sort is an introsort whose tie order is fixed by its algorithm: ties come
// out in index order only below 17 elements, where it is a plain insertion sort.  The functions below follow libstdc++'s
// __introsort_loop / __final_insertion_sort / __partial_sort step for step, so equal scores end in the order the reference
// sees.  One thread runs it on shared memory.
struct SortView {
  float* key;
  int* idx;
  __device__ __forceinline__ bool less(int a, int b) const { return key[a] > key[b]; }  // comp(*a, *b)
  __device__ __forceinline__ void swap(int a, int b) const {
    const float k = key[a];
    key[a] = key[b];
    key[b] = k;
    const int i = idx[a];
    idx[a] = idx[b];
    idx[b] = i;
  }
  __device__ __forceinline__ void move(int dst, int src) const {
    key[dst] = key[src];
    idx[dst] = idx[src];
  }
};

__device__ void push_heap(const SortView& s, int first, int hole, int top, float vk, int vi) {
  int parent = (hole - 1) / 2;
  while (hole > top && s.key[first + parent] > vk) {
    s.move(first + hole, first + parent);
    hole = parent;
    parent = (hole - 1) / 2;
  }
  s.key[first + hole] = vk;
  s.idx[first + hole] = vi;
}

__device__ void adjust_heap(const SortView& s, int first, int hole, int len, float vk, int vi) {
  const int top = hole;
  int child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (s.less(first + child, first + child - 1)) child--;
    s.move(first + hole, first + child);
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    s.move(first + hole, first + child - 1);
    hole = child - 1;
  }
  push_heap(s, first, hole, top, vk, vi);
}

// __partial_sort(first, last, last): __make_heap then __sort_heap
__device__ void heap_sort(const SortView& s, int first, int last) {
  const int len = last - first;
  if (len >= 2) {
    for (int parent = (len - 2) / 2;; --parent) {
      adjust_heap(s, first, parent, len, s.key[first + parent], s.idx[first + parent]);
      if (parent == 0) break;
    }
  }
  while (last - first > 1) {
    --last;
    const float vk = s.key[last];
    const int vi = s.idx[last];
    s.move(last, first);
    adjust_heap(s, first, 0, last - first, vk, vi);
  }
}

__device__ void unguarded_linear_insert(const SortView& s, int last) {
  const float vk = s.key[last];
  const int vi = s.idx[last];
  int next = last - 1;
  while (vk > s.key[next]) {
    s.move(last, next);
    last = next;
    --next;
  }
  s.key[last] = vk;
  s.idx[last] = vi;
}

__device__ void insertion_sort(const SortView& s, int first, int last) {
  if (first == last) return;
  for (int i = first + 1; i != last; ++i) {
    if (s.less(i, first)) {
      const float vk = s.key[i];
      const int vi = s.idx[i];
      for (int j = i; j > first; --j) s.move(j, j - 1);
      s.key[first] = vk;
      s.idx[first] = vi;
    } else {
      unguarded_linear_insert(s, i);
    }
  }
}

__device__ void std_sort(const SortView& s, int n) {
  constexpr int kThreshold = 16;
  if (n <= 1) return;
  // __introsort_loop: the recursion on [cut, last) becomes a stack; the disjoint ranges are sorted independently, so the order
  // they are visited in does not change the result
  int st_first[32], st_last[32], st_depth[32];  // at most 2 * lg(4096) + 1 = 25 pending ranges
  int top = 0;
  st_first[0] = 0;
  st_last[0] = n;
  st_depth[0] = 2 * (31 - __clz(n));  // 2 * std::__lg(n)
  top = 1;
  while (top > 0) {
    --top;
    int first = st_first[top], last = st_last[top], depth = st_depth[top];
    while (last - first > kThreshold) {
      if (depth == 0) {
        heap_sort(s, first, last);
        break;
      }
      --depth;
      // __unguarded_partition_pivot: __move_median_to_first(first, first + 1, mid, last - 1), then partition [first + 1, last)
      const int a = first + 1, b = first + (last - first) / 2, c = last - 1;
      int m;
      if (s.less(a, b)) {
        m = s.less(b, c) ? b : (s.less(a, c) ? c : a);
      } else {
        m = s.less(a, c) ? a : (s.less(b, c) ? c : b);
      }
      s.swap(first, m);
      int lo = first + 1, hi = last;
      while (true) {
        while (s.less(lo, first)) ++lo;
        --hi;
        while (s.less(first, hi)) --hi;
        if (!(lo < hi)) break;
        s.swap(lo, hi);
        ++lo;
      }
      st_first[top] = lo;
      st_last[top] = last;
      st_depth[top] = depth;
      ++top;
      last = lo;
    }
  }
  // __final_insertion_sort
  if (n > kThreshold) {
    insertion_sort(s, 0, kThreshold);
    for (int i = kThreshold; i < n; ++i) unguarded_linear_insert(s, i);
  } else {
    insertion_sort(s, 0, n);
  }
}

// float -> unsigned key with the same order (finite values; -0 and +0 equal)
__device__ __forceinline__ uint32_t order_key(float x) {
  uint32_t u = __float_as_uint(x);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

struct HlTopkArgs {
  const float* scores;     // [V, S]
  const int32_t* n_score;  // [V]
  const int32_t* n_cut;    // [V]
  const float* labels;     // [V, C, A]
  const int32_t* n_label;  // [V]
  double* ap;              // [V, A]
  int V, S, C, A, median;
};

__global__ void __launch_bounds__(kMaxAnno * 32) eval_hl_topk_kernel(const HlTopkArgs a) {
  pdl_prologue();
  __shared__ float s_key[kMaxClips];
  __shared__ int s_idx[kMaxClips];
  __shared__ float s_thr[kMaxAnno];
  const int v = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int n = a.n_score[v], nc = a.n_cut[v], nl = a.n_label[v];
  const float* lab = a.labels + (size_t)v * a.C * a.A + w;  // column w, stride A
  for (int i = tid; i < n; i += blockDim.x) {
    s_key[i] = a.scores[(size_t)v * a.S + i];
    s_idx[i] = i;
  }
  // threshold of annotator w: torch's median (the lower one) of the whole label column, or 0
  float thr = 0.0f;
  if (a.median) {
    const int rank = (nl - 1) / 2;  // the (rank+1)-th smallest value: the smallest key K with #(key <= K) > rank
    uint32_t lo = 0u, hi = 0xffffffffu;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      int cnt = 0;
      for (int i = lane; i < nl; i += 32) cnt += order_key(lab[(size_t)i * a.A]) <= mid;
#pragma unroll
      for (int off = 16; off; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
      if (cnt > rank) hi = mid;
      else lo = mid + 1;
    }
    thr = key_value(lo);
  }
  if (lane == 0) s_thr[w] = thr;
  __syncthreads();
  if (tid == 0) std_sort(SortView{s_key, s_idx}, n);
  __syncthreads();

  // AP of annotator w over the first nc sorted clips.  The reference's recursion adds 0 at a negative clip, and at a positive
  // clip j (hits h0 before it, h1 = h0 + 1 after) it adds ((h1/ngt - h0/ngt) * (prc + h1/(j+1))) / 2 with prc = h0/j (1 at
  // j = 0): every term is computed in parallel, the sum runs left to right in lane 0.
  thr = s_thr[w];
  int ngt = 0;
  for (int base = 0; base < nc; base += 32) {
    const int j = base + lane;
    ngt += __popc(__ballot_sync(0xffffffffu, j < nc && lab[(size_t)s_idx[j] * a.A] > thr));
  }
  double ap = 0.0;
  if (ngt > 0) {
    const double dn = (double)ngt;
    int carry = 0;
    for (int base = 0; base < nc; base += 32) {
      const int j = base + lane;
      const bool pos = j < nc && lab[(size_t)s_idx[j] * a.A] > thr;
      const unsigned ball = __ballot_sync(0xffffffffu, pos);
      const int h1 = carry + __popc(ball & ((2u << lane) - 1u)), h0 = h1 - (int)pos;
      double term = 0.0;
      if (pos) {
        const double rec = __ddiv_rn((double)h0, dn), rec1 = __ddiv_rn((double)h1, dn);
        const double prc = j == 0 ? 1.0 : __ddiv_rn((double)h0, (double)j);
        const double prc1 = __ddiv_rn((double)h1, (double)(j + 1));
        term = __ddiv_rn(__dmul_rn(__dsub_rn(rec1, rec), __dadd_rn(prc, prc1)), 2.0);
      }
      for (int t = 0; t < 32; ++t) {
        const double x = __shfl_sync(0xffffffffu, term, t);
        if ((ball >> t) & 1u) ap = __dadd_rn(ap, x);
      }
      carry += __popc(ball);
    }
  }
  if (lane == 0) a.ap[(size_t)v * a.A + w] = ap;
}

// ---- maximum-weight bipartite matching ---------------------------------------------------------------------------------
// W[i, j] = |a_i & b_j| / |a_i | b_j| (0 for two empty tag sets), generated from the 64-bit tag masks whenever it is read.
__device__ __forceinline__ double semantic_iou(uint64_t x, uint64_t y) {
  const int u = __popcll(x | y);
  return u ? __ddiv_rn((double)__popcll(x & y), (double)u) : 0.0;
}

struct MatchArgs {
  const uint64_t* a;      // machine-summary tag masks, queries concatenated
  const int32_t* a_off;   // [Q + 1]
  const uint64_t* b;      // ground-truth-summary tag masks
  const int32_t* b_off;   // [Q + 1]
  double* s;              // [Q]
  int max_side;
};

// smaller (value, column) first
__device__ __forceinline__ void argmin_merge(double& v, int& j, double ov, int oj) {
  if (ov < v || (ov == v && (unsigned)oj < (unsigned)j)) {
    v = ov;
    j = oj;
  }
}

// Hungarian method with shortest augmenting paths (potentials u, v in fp64) on the cost -W, rows = the smaller side.  Row r
// is inserted through a virtual column (index m); each step scans the columns not yet on the alternating tree (one thread per
// column group, a block argmin picks the next one), so a row needs at most m steps and the total is O(n^2 m) in the worst case.
__global__ void __launch_bounds__(kMatchThreads) qfvs_match_kernel(const MatchArgs a) {
  pdl_prologue();
  __shared__ uint64_t s_row[kMaxSide];
  __shared__ double s_u[kMaxSide];
  __shared__ int s_p[kMaxSide + 1];  // s_p[j]: row on column j, -1 when free; s_p[m]: the row being inserted
  __shared__ int s_way[kMaxSide];
  __shared__ double s_rv[kMatchThreads / 32];
  __shared__ int s_rj[kMatchThreads / 32];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  const uint64_t* A = a.a + a.a_off[q];
  const uint64_t* B = a.b + a.b_off[q];
  int na = a.a_off[q + 1] - a.a_off[q], nb = a.b_off[q + 1] - a.b_off[q];
  const bool swap = na > nb;  // W is symmetric in its arguments: match the smaller side into the larger
  const uint64_t* R = swap ? B : A;
  const uint64_t* Cm = swap ? A : B;
  const int n = swap ? nb : na, m = swap ? na : nb;
  if (n < 1 || m > a.max_side) {  // a side outside 1..max_side: NaN (the host checks both sides before the launch)
    if (tid == 0) a.s[q] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  uint64_t cm[kColsPerThread];
  double vpot[kColsPerThread], minv[kColsPerThread];
#pragma unroll
  for (int t = 0; t < kColsPerThread; ++t) {
    const int j = tid + t * kMatchThreads;
    cm[t] = j < m ? Cm[j] : 0ull;
    vpot[t] = 0.0;
    if (j < m) s_p[j] = -1;
  }
  for (int i = tid; i < n; i += kMatchThreads) {
    s_row[i] = R[i];
    s_u[i] = 0.0;
  }
  __syncthreads();
  for (int r = 0; r < n; ++r) {
    if (tid == 0) s_p[m] = r;
    unsigned used = 0;
#pragma unroll
    for (int t = 0; t < kColsPerThread; ++t) minv[t] = INFINITY;
    int j0 = m;
    __syncthreads();
    while (true) {
      if (j0 < m && j0 % kMatchThreads == tid) used |= 1u << (j0 / kMatchThreads);
      const int i0 = s_p[j0];
      const double ui = s_u[i0];
      const uint64_t rm = s_row[i0];
      double best = INFINITY;
      int bj = -1;
#pragma unroll
      for (int t = 0; t < kColsPerThread; ++t) {
        const int j = tid + t * kMatchThreads;
        if (j < m && !((used >> t) & 1u)) {
          const double cur = __dsub_rn(__dsub_rn(-semantic_iou(rm, cm[t]), ui), vpot[t]);
          if (cur < minv[t]) {
            minv[t] = cur;
            s_way[j] = j0;
          }
          argmin_merge(best, bj, minv[t], j);
        }
      }
#pragma unroll
      for (int off = 16; off; off >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, best, off);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, off);
        argmin_merge(best, bj, ov, oj);
      }
      if (lane == 0) {
        s_rv[wp] = best;
        s_rj[wp] = bj;
      }
      __syncthreads();
      double delta = s_rv[0];
      int j1 = s_rj[0];
      for (int k = 1; k < kMatchThreads / 32; ++k) argmin_merge(delta, j1, s_rv[k], s_rj[k]);
      // decided before the barrier below: s_p does not change inside this loop, but thread 0 rewrites it in the path flip as
      // soon as it leaves, so no thread may read it after that barrier
      const bool free_col = s_p[j1] < 0;
#pragma unroll
      for (int t = 0; t < kColsPerThread; ++t) {
        const int j = tid + t * kMatchThreads;
        if (j < m) {
          if ((used >> t) & 1u) {
            s_u[s_p[j]] = __dadd_rn(s_u[s_p[j]], delta);
            vpot[t] = __dsub_rn(vpot[t], delta);
          } else {
            minv[t] = __dsub_rn(minv[t], delta);
          }
        }
      }
      if (tid == 0) s_u[r] = __dadd_rn(s_u[r], delta);  // the virtual column, always on the tree
      __syncthreads();
      j0 = j1;
      if (free_col) break;
    }
    if (tid == 0) {  // flip the alternating path ending at the free column j0
      while (j0 != m) {
        const int j1 = s_way[j0];
        s_p[j0] = s_p[j1];
        j0 = j1;
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    double s = 0.0;
    for (int j = 0; j < m; ++j)
      if (s_p[j] >= 0) s = __dadd_rn(s, semantic_iou(s_row[s_p[j]], Cm[j]));
    a.s[q] = s;
  }
}

// ---- QFVS evaluation epoch: per-query score, top k and the matching's machine side --------------------------------------
// main/inference_qfvs.py eval_epoch for the queries of one chunk: the score of each kept position in the reference's fp32
// order, score.topk(k) as torch.topk on CUDA orders it (descending, NaN above every number; ties by ascending index above 32
// results, by torch's bitonic network up to 32) and the
// tag masks of the chosen shots.  One block per query; the top k comes from a bitonic sort of n (<= 8,192) 64-bit keys
// (order-preserving score << 32 | ~index) in shared memory.
constexpr int kSelectMaxN = 8192;
constexpr int kSelectThreads = 1024;
constexpr int kTopkSmallSort = 32;  // torch.topk results up to this size are sorted by at::native's unstable bitonic network

struct SelectArgs {
  const float* logits[3];  // [F, N] per variant: concept 1, concept 2, both (NULL when the variant is not read)
  const float* sal[3];
  const int32_t* pos;      // [n] kept positions of mask_GT, row-major, cut to n
  const uint64_t* tags;    // [>= n] tag mask per shot
  float* score;            // [Q, n]
  int32_t* top;            // [Q, k]
  uint64_t* a;             // [Q, k]
  int N, n, k, mode, gather, q0;
};

__device__ __forceinline__ float variant_score(const SelectArgs& a, int v, size_t i) {
  if (a.mode == 0) return a.logits[v][i];
  if (a.mode == 1) return a.sal[v][i];
  return __fadd_rn(__fadd_rn(0.0f, a.logits[v][i]), a.sal[v][i]);  // torch.zeros(n) += pred_logits; += saliency_scores
}

// descending order of torch.topk: NaN first, -0 == +0
__device__ __forceinline__ uint32_t topk_key(float x) { return isnan(x) ? 0xffffffffu : order_key(x); }

__global__ void __launch_bounds__(kSelectThreads) qfvs_eval_select_kernel(const SelectArgs a) {
  pdl_prologue();
  extern __shared__ unsigned long long s_key[];
  const int f = blockIdx.x, tid = threadIdx.x;
  const size_t q = (size_t)a.q0 + f;
  int P = 1;
  while (P < a.n) P <<= 1;
  for (int i = tid; i < P; i += kSelectThreads) {
    unsigned long long key = 0ull;  // below every real key: order_key(-inf) = 0x007fffff
    if (i < a.n) {
      const size_t p = (size_t)f * a.N + a.pos[i];
      float s = variant_score(a, 2, p);
      if (a.gather) s = __fadd_rn(__fadd_rn(s, variant_score(a, 0, p)), variant_score(a, 1, p));  // score + score1 + score2
      a.score[q * a.n + i] = s;
      key = ((unsigned long long)topk_key(s) << 32) | (uint32_t)~(uint32_t)i;
    }
    s_key[i] = key;
  }
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = tid; t < P / 2; t += kSelectThreads) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const unsigned long long x = s_key[lo], y = s_key[hi];
        if (((lo & size) == 0) == (x < y)) {  // blocks with (lo & size) == 0 run descending, so the last pass is descending
          s_key[lo] = y;
          s_key[hi] = x;
        }
      }
      __syncthreads();
    }
  }
  if (a.k > kTopkSmallSort) {  // torch.topk sorts larger results stably: ties stay in ascending index order
    for (int j = tid; j < a.k; j += kSelectThreads) {
      const int i = (int)~(uint32_t)s_key[j];
      a.top[q * a.k + j] = i;
      a.a[q * a.k + j] = a.tags[i];
    }
    return;
  }
  // k <= 32: torch.topk gathers the chosen elements (those above the k-th score by ascending index, then those equal to it by
  // ascending index) and sorts them with a 32-wide bitonic network that is not stable; warp 0 runs the same network
  __shared__ unsigned long long s_small[kTopkSmallSort];  // (score key << 32) | index
  __shared__ bool s_valid[kTopkSmallSort];
  if (tid >= 32) return;
  const int lane = tid;
  const uint32_t kth = (uint32_t)(s_key[a.k - 1] >> 32);
  const unsigned long long e = lane < a.k ? s_key[lane] : 0ull;
  const uint32_t hi = (uint32_t)(e >> 32), idx = ~(uint32_t)e;
  const bool above = lane < a.k && hi > kth;
  const unsigned above_mask = __ballot_sync(0xffffffffu, above);
  int before = 0;  // entries above the k-th score with a smaller index
  for (int j = 0; j < 32; ++j) {
    const uint32_t other = __shfl_sync(0xffffffffu, idx, j);
    before += ((above_mask >> j) & 1u) && other < idx;
  }
  const int slot = above ? before : lane;  // the equal ones already sit at the end of the first k, by ascending index
  s_small[slot] = lane < a.k ? (((unsigned long long)hi << 32) | idx) : 0ull;
  s_valid[slot] = lane < a.k;
  __syncwarp();
  // at::native bitonicSort<32> with GTOp: swap = (A > B && validA) || !validB; exchange when swap == dir
  auto step = [&](int stride, bool dir) {
    if (lane < kTopkSmallSort / 2) {
      const int p = 2 * lane - (lane & (stride - 1)), r = p + stride;
      const bool sw = ((uint32_t)(s_small[p] >> 32) > (uint32_t)(s_small[r] >> 32) && s_valid[p]) || !s_valid[r];
      if (sw == dir) {
        const unsigned long long t = s_small[p];
        s_small[p] = s_small[r];
        s_small[r] = t;
        const bool v = s_valid[p];
        s_valid[p] = s_valid[r];
        s_valid[r] = v;
      }
    }
    __syncwarp();
  };
  for (int size = 2; size < kTopkSmallSort; size *= 2)
    for (int stride = size / 2; stride > 0; stride /= 2) step(stride, (lane & (size / 2)) != 0);
  for (int stride = kTopkSmallSort / 2; stride > 0; stride /= 2) step(stride, false);
  if (lane < a.k) {
    const int i = (int)(uint32_t)s_small[lane];
    a.top[q * a.k + lane] = i;
    a.a[q * a.k + lane] = a.tags[i];
  }
}

}  // namespace
}  // namespace uv

extern "C" int univtg_eval_hl_topk(const float* scores, const int32_t* n_score, const int32_t* n_cut, const float* labels,
                                   const int32_t* n_label, int32_t V, int32_t S, int32_t C, int32_t A, int32_t median, double* ap,
                                   void* stream) {
  using namespace uv;
  if (!scores || !n_score || !n_cut || !labels || !n_label || !ap || V < 0 || S < 1 || S > kMaxClips || C < 1 || C > kMaxClips ||
      A < 1 || A > kMaxAnno || (median != 0 && median != 1)) {
    set_error("univtg_eval_hl_topk: bad argument (S and C must be in 1..%d, A in 1..%d, median 0 or 1)", kMaxClips, kMaxAnno);
    return 1;
  }
  if (V == 0) return 0;
  HlTopkArgs args{scores, n_score, n_cut, labels, n_label, ap, V, S, C, A, median};
  launch_k(eval_hl_topk_kernel, dim3(V), dim3(32 * A), 0, reinterpret_cast<cudaStream_t>(stream), args);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_eval_hl_topk launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

extern "C" int univtg_qfvs_match(const uint64_t* a, const int32_t* a_off, const uint64_t* b, const int32_t* b_off, int32_t Q,
                                 int32_t max_side, double* s, void* stream) {
  using namespace uv;
  if (!a || !a_off || !b || !b_off || !s || Q < 0 || max_side < 1 || max_side > kMaxSide) {
    set_error("univtg_qfvs_match: bad argument (max_side must be in 1..%d)", kMaxSide);
    return 1;
  }
  if (Q == 0) return 0;
  MatchArgs args{a, a_off, b, b_off, s, max_side};
  launch_k(qfvs_match_kernel, dim3(Q), dim3(kMatchThreads), 0, reinterpret_cast<cudaStream_t>(stream), args);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_qfvs_match launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

extern "C" int univtg_qfvs_eval_select(const float* logits1, const float* sal1, const float* logits2, const float* sal2,
                                       const float* logits_o, const float* sal_o, const int32_t* pos, const uint64_t* tags, int32_t F,
                                       int32_t N, int32_t n, int32_t k, int32_t mode, int32_t gather, int32_t q0, float* score,
                                       int32_t* top, uint64_t* a, void* stream) {
  using namespace uv;
  const bool need_l = mode != 1, need_s = mode != 0;
  bool ok = pos && tags && score && top && a && F >= 0 && N >= 1 && n >= 1 && n <= N && n <= kSelectMaxN && k >= 1 && k <= n &&
            mode >= 0 && mode <= 2 && (gather == 0 || gather == 1) && q0 >= 0;
  const float* lg[3] = {logits1, logits2, logits_o};
  const float* sl[3] = {sal1, sal2, sal_o};
  for (int v = gather ? 0 : 2; ok && v < 3; ++v) ok = (!need_l || lg[v]) && (!need_s || sl[v]);
  if (!ok) {
    set_error("univtg_qfvs_eval_select: bad argument (n in 1..min(N, %d), k in 1..n, mode 0..2, gather 0 or 1, the outputs the "
              "mode and gather read non-NULL)", kSelectMaxN);
    return 1;
  }
  if (F == 0) return 0;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(qfvs_eval_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kSelectMaxN * (int)sizeof(unsigned long long));
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(qfvs_eval_select): %s", cudaGetErrorString(e));
      return (int)e;
    }
    attr_set = true;
  }
  int P = 1;
  while (P < n) P <<= 1;
  SelectArgs args{{logits1, logits2, logits_o}, {sal1, sal2, sal_o}, pos, tags, score, top, a, N, n, k, mode, gather, q0};
  launch_k(qfvs_eval_select_kernel, dim3(F), dim3(kSelectThreads), (size_t)P * sizeof(unsigned long long),
           reinterpret_cast<cudaStream_t>(stream), args);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("univtg_qfvs_eval_select launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}
