// Post-forward decode of the reference's moment-retrieval evaluation loop, on the device (SURVEY.md section 8 rows a16 and f-1):
//   main/inference_mr.py:112-120  scores = pred_logits[..., 0]; pred_spans = timestamp + pred_spans; scores[~timestamp_mask] = 0
//   main/inference_mr.py:146-157  spans * duration, clamp(0, duration), rows [st, ed, score] sorted by score (descending, Python's
//                                 stable sort: ties keep clip order), every number then rounded like float(f"{e:.4f}")
//   main_gradio.py:100-106        same windows in clip units; top-1 / top-k are the first rows of the sorted list
//   utils/temporal_nms.py:25-74   greedy temporal NMS on the rounded (double) rows, "IoU" = intersection / convex hull
//   main/inference_mr.py:122-136  highlight values: fp16(saliency), or with eval_mode "add" fp32(fp16(saliency)) + prob
//   eval/postprocessing.py:26-51  round_multiple: windows snapped to multiples of clip_length in fp32, score re-rounded
// The epoch path (univtg_decode_mr_pool / univtg_temporal_nms_pool) writes every batch into one ragged row pool at a row offset
// and runs the NMS of the whole epoch in one launch.
// All of it is HBM-trivial integer/compare work: one block per sample, a bitonic sort in shared memory, exact integer
// arithmetic for the decimal rounding, IEEE double for the NMS so that every keep/suppress decision equals the Python code's.
#include <math.h>
#include <stdint.h>

#include "../../include/univtg_b200.h"
#include "kernels.h"
#include "ptx.cuh"

namespace uv {
namespace {

// float(f"{e:.4f}") for a float32 e: the nearest double to the decimal obtained by rounding e's EXACT binary value to four
// decimals, ties to even (what printf does).  e = m * 2^x with a 24-bit m, so m * 10^4 fits 38 bits: the rounding is exact
// integer arithmetic, and k / 1e4 (correctly rounded division) is the double Python parses from the decimal string.
__device__ __forceinline__ double round4_like_python(float f) {
  const uint32_t bits = __float_as_uint(f);
  const uint32_t ex = (bits >> 23) & 0xff;
  const bool neg = (bits >> 31) != 0;
  if (ex == 0xff) return (double)f;  // inf / nan: pass through
  uint64_t m = bits & 0x7fffff;
  int x;
  if (ex == 0) {
    x = -149;  // subnormal
  } else {
    m |= 0x800000;
    x = (int)ex - 150;
  }
  uint64_t k;
  const uint64_t P = m * 10000ull;
  if (x >= 0) {
    if (x > 20) return (double)f;  // >= 2^44: already an integer far beyond four decimals of interest
    k = P << x;
  } else {
    const int s = -x;
    if (s > 62) {
      k = 0;
    } else {
      const uint64_t q = P >> s, r = P & ((1ull << s) - 1), half = 1ull << (s - 1);
      k = q + ((r > half || (r == half && (q & 1))) ? 1 : 0);
    }
  }
  const double v = __ddiv_rn((double)k, 10000.0);
  return neg ? -v : v;
}

struct DecodeArgs {
  const float* logits;     // [B, Lv] (pred_logits[..., 0])
  const float* spans;      // [B, Lv, 2]
  const float* timestamp;  // [B, Lv, 2]
  const float* tmask;      // [B, Lv]
  const float* duration;   // [B] or null (1.0: windows stay in the units of timestamp)
  const float* saliency;   // [B, Lv] or null (no highlight values)
  const float* vid_mask;   // [B, Lv] or null (no valid lengths)
  float* windows;          // [B, Lv, 3] or null
  double* windows_r4;      // [B, Lv, 3] or null
  int32_t* order;          // [B, Lv] or null
  float* hl;               // [B, Lv], written when saliency != null
  int32_t* valid_len;      // [B], written when vid_mask != null
  int B, Lv, npad, sort;
  int add_prob;            // eval_mode == "add": hl = fp32(fp16(saliency)) + prob
  int round_multiple;      // > 0: PostProcessorDETR.round_to_multiple_clip_lengths on the rounded rows
  float clip_length;
};

// torch.round(windows / clip_length) * clip_length on a float32 tensor: IEEE division (not a reciprocal multiply), round half to
// even, fp32 product; the result is widened to double by .tolist().
__device__ __forceinline__ double round_to_clip_multiple(double r4, float clip) {
  return (double)__fmul_rn(rintf(__fdiv_rn(__double2float_rn(r4), clip)), clip);
}

// (score, index) keys; a precedes b when its score is larger, ties by smaller clip index (== Python's stable descending sort)
__device__ __forceinline__ bool precedes(float sa, int ia, float sb, int ib) { return sa > sb || (sa == sb && ia < ib); }

__global__ void __launch_bounds__(256) decode_mr_kernel(const DecodeArgs a) {
  pdl_prologue();
  extern __shared__ uint8_t sm_raw[];
  float* s_key = reinterpret_cast<float*>(sm_raw);          // [npad]
  int* s_idx = reinterpret_cast<int*>(s_key + a.npad);      // [npad]
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  if (a.saliency) {
    // _saliency_scores[b, i]: saliency.half() (+ prob, where prob[..., 0] is 0 at masked clips after scores[~mask] = 0)
    for (int i = tid; i < a.Lv; i += nt) {
      const size_t k = (size_t)b * a.Lv + i;
      float v = __half2float(__float2half_rn(a.saliency[k]));
      if (a.add_prob) v = __fadd_rn(v, a.tmask[k] == 0.f ? 0.f : a.logits[k]);
      a.hl[k] = v;
    }
  }
  if (a.vid_mask && tid < 32) {  // src_vid_mask.sum(1): the number of valid clips (0 / 1 masks sum exactly in fp32)
    float acc = 0.f;
    for (int i = tid; i < a.Lv; i += 32) acc += a.vid_mask[(size_t)b * a.Lv + i];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (tid == 0) a.valid_len[b] = (int32_t)acc;
  }
  for (int i = tid; i < a.npad; i += nt) {
    float sc = -INFINITY;  // padding sorts last
    if (i < a.Lv) {
      sc = a.logits[(size_t)b * a.Lv + i];
      if (a.tmask[(size_t)b * a.Lv + i] == 0.f) sc = 0.f;  // scores[~mask] = 0
    }
    s_key[i] = sc;
    s_idx[i] = i;
  }
  __syncthreads();
  if (a.sort) {
    for (int k = 2; k <= a.npad; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < a.npad; i += nt) {
          const int p = i ^ j;
          if (p > i) {
            const bool up = (i & k) == 0;  // this pair ends with the "earlier" element at i
            const float si = s_key[i], sp = s_key[p];
            const int ii = s_idx[i], ip = s_idx[p];
            const bool swap = up ? precedes(sp, ip, si, ii) : precedes(si, ii, sp, ip);
            if (swap) {
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
  }
  const float dur = a.duration ? a.duration[b] : 1.0f;
  for (int r = tid; r < a.Lv; r += nt) {
    const int i = s_idx[r];
    const size_t src = ((size_t)b * a.Lv + i) * 2;
    // fp32, same operation order as the reference: (timestamp + pred_spans) * duration, clamp to [0, duration]
    float st = (a.timestamp[src] + a.spans[src]) * dur;
    float ed = (a.timestamp[src + 1] + a.spans[src + 1]) * dur;
    if (a.duration) {
      st = fminf(fmaxf(st, 0.f), dur);
      ed = fminf(fmaxf(ed, 0.f), dur);
    }
    const float sc = s_key[r];
    const size_t o = ((size_t)b * a.Lv + r) * 3;
    if (a.windows) {
      a.windows[o] = st;
      a.windows[o + 1] = ed;
      a.windows[o + 2] = sc;
    }
    if (a.windows_r4) {
      double r4_st = round4_like_python(st), r4_ed = round4_like_python(ed), r4_sc = round4_like_python(sc);
      if (a.round_multiple > 0) {  // torch.tensor(rows) is fp32; the score column is only re-rounded: float(f"{e[2]:.4f}")
        r4_st = round_to_clip_multiple(r4_st, a.clip_length);
        r4_ed = round_to_clip_multiple(r4_ed, a.clip_length);
        r4_sc = round4_like_python(__double2float_rn(r4_sc));
      }
      a.windows_r4[o] = r4_st;
      a.windows_r4[o + 1] = r4_ed;
      a.windows_r4[o + 2] = r4_sc;
    }
    if (a.order) a.order[(size_t)b * a.Lv + r] = i;
  }
}

struct NmsArgs {
  const double* windows;  // [B, n, 3] sorted by score (descending), or the row pool when offsets != null
  const int64_t* offsets; // [B + 1] or null: sample b owns pool rows offsets[b] .. offsets[b + 1] - 1
  double* out;            // [B, max_after, 3]
  int32_t* counts;        // [B]
  double thd;
  int B, n, n_in, max_before, max_after;
  int sort;               // sort the first rows by score first (stable, descending), as temporal_nms does
};

// utils/temporal_nms.py: intersection / (max end - min start); 0 when the hull is empty.  IEEE double, no contraction.
__device__ __forceinline__ double hull_iou(double s0, double e0, double s1, double e1) {
  const double inter = fmax(0.0, fmin(e0, e1) - fmax(s0, s1));
  const double uni = fmax(e0, e1) - fmin(s0, s1);
  if (uni == 0.0) return 0.0;
  return __ddiv_rn(inter, uni);
}

__global__ void __launch_bounds__(128) temporal_nms_kernel(const NmsArgs a) {
  pdl_prologue();
  extern __shared__ uint8_t sm_raw[];
  double* s_st = reinterpret_cast<double*>(sm_raw);  // [n_in]
  double* s_ed = s_st + a.n_in;
  double* s_sc = s_ed + a.n_in;
  int* s_alive = reinterpret_cast<int*>(s_sc + a.n_in);
  const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const double* w = a.windows + (a.offsets ? (size_t)a.offsets[b] : (size_t)b * a.n) * 3;
  int n_in = a.n_in;
  if (a.offsets) {
    const int64_t rows = a.offsets[b + 1] - a.offsets[b];
    n_in = rows < a.max_before ? (int)rows : a.max_before;
  }
  if (a.sort) {
    // sorted(rows[:max_before], key=score, reverse=True): row i goes to the number of rows that precede it
    for (int i = tid; i < n_in; i += nt) s_sc[i] = w[3 * i + 2];
    __syncthreads();
    for (int i = tid; i < n_in; i += nt) {
      const double si = s_sc[i];
      int rank = 0;
      for (int j = 0; j < n_in; ++j) rank += (s_sc[j] > si || (s_sc[j] == si && j < i)) ? 1 : 0;
      s_alive[i] = rank;
    }
    __syncthreads();
    for (int i = tid; i < n_in; i += nt) {
      const int r = s_alive[i];
      s_st[r] = w[3 * i];
      s_ed[r] = w[3 * i + 1];
      s_sc[r] = w[3 * i + 2];
    }
    __syncthreads();
    for (int i = tid; i < n_in; i += nt) s_alive[i] = 1;
  } else {
    for (int i = tid; i < n_in; i += nt) {
      s_st[i] = w[3 * i];
      s_ed[i] = w[3 * i + 1];
      s_sc[i] = w[3 * i + 2];
      s_alive[i] = 1;
    }
  }
  __syncthreads();
  int kept = 0;
  for (int i = 0; i < n_in && kept < a.max_after; ++i) {
    if (!s_alive[i]) continue;  // block-uniform (shared flag, read after a barrier)
    if (tid == 0) {
      double* o = a.out + ((size_t)b * a.max_after + kept) * 3;
      o[0] = s_st[i];
      o[1] = s_ed[i];
      o[2] = s_sc[i];
    }
    ++kept;
    const double s0 = s_st[i], e0 = s_ed[i];
    for (int j = i + 1 + tid; j < n_in; j += nt)
      if (s_alive[j] && hull_iou(s0, e0, s_st[j], s_ed[j]) > a.thd) s_alive[j] = 0;
    __syncthreads();
  }
  if (tid == 0) a.counts[b] = kept;
}

}  // namespace
}  // namespace uv

namespace uv {
namespace {

// npad = Lv rounded up to a power of two (the bitonic sort's width), or 0 when Lv > 4096
int decode_npad(int Lv) {
  int npad = 1;
  while (npad < Lv) npad <<= 1;
  return npad > 4096 ? 0 : npad;
}

int launch_decode(const DecodeArgs& a, void* stream, const char* what) {
  launch_k(decode_mr_kernel, dim3(a.B), dim3(256), (size_t)a.npad * 8, reinterpret_cast<cudaStream_t>(stream), a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("%s launch failed: %s", what, cudaGetErrorString(e));
  return (int)e;
}

int launch_nms(const NmsArgs& a, void* stream, const char* what) {
  launch_k(temporal_nms_kernel, dim3(a.B), dim3(128), (size_t)a.n_in * 28 + 8, reinterpret_cast<cudaStream_t>(stream), a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("%s launch failed: %s", what, cudaGetErrorString(e));
  return (int)e;
}

}  // namespace
}  // namespace uv

extern "C" int univtg_decode_mr(const float* pred_logits, const float* pred_spans, const float* timestamp, const float* timestamp_mask,
                                const float* duration, int32_t B, int32_t Lv, int32_t sort, float* windows, double* windows_r4,
                                int32_t* order, void* stream) {
  using namespace uv;
  if (!pred_logits || !pred_spans || !timestamp || !timestamp_mask || !windows || B < 0 || Lv < 1) {
    set_error("univtg_decode_mr: bad argument");
    return 1;
  }
  if (B == 0) return 0;
  const int npad = decode_npad(Lv);
  if (!npad) {
    set_error("univtg_decode_mr: Lv %d > 4096 not supported", Lv);
    return 1;
  }
  DecodeArgs a;
  memset(&a, 0, sizeof(a));
  a.logits = pred_logits;
  a.spans = pred_spans;
  a.timestamp = timestamp;
  a.tmask = timestamp_mask;
  a.duration = duration;
  a.windows = windows;
  a.windows_r4 = windows_r4;
  a.order = order;
  a.B = B;
  a.Lv = Lv;
  a.npad = npad;
  a.sort = sort;
  return launch_decode(a, stream, "univtg_decode_mr");
}

extern "C" int univtg_decode_mr_pool(const float* pred_logits, const float* pred_spans, const float* timestamp,
                                     const float* timestamp_mask, const float* duration, const float* saliency_scores,
                                     const float* src_vid_mask, int32_t B, int32_t Lv, int32_t sort, int32_t add_prob,
                                     int32_t round_multiple, float clip_length, int64_t row_offset, int64_t sample_offset, double* rows,
                                     float* hl, int32_t* valid_len, void* stream) {
  using namespace uv;
  if (!pred_logits || !pred_spans || !timestamp || !timestamp_mask || !rows || B < 0 || Lv < 1 || row_offset < 0 ||
      sample_offset < 0 || (saliency_scores && !hl) || (src_vid_mask && !valid_len) || (add_prob && !saliency_scores) ||
      (round_multiple > 0 && !(clip_length > 0.f))) {
    set_error("univtg_decode_mr_pool: bad argument");
    return 1;
  }
  if (B == 0) return 0;
  const int npad = decode_npad(Lv);
  if (!npad) {
    set_error("univtg_decode_mr_pool: Lv %d > 4096 not supported", Lv);
    return 1;
  }
  DecodeArgs a;
  memset(&a, 0, sizeof(a));
  a.logits = pred_logits;
  a.spans = pred_spans;
  a.timestamp = timestamp;
  a.tmask = timestamp_mask;
  a.duration = duration;
  a.saliency = saliency_scores;
  a.vid_mask = src_vid_mask;
  a.windows_r4 = rows + row_offset * 3;
  a.hl = saliency_scores ? hl + row_offset : nullptr;
  a.valid_len = src_vid_mask ? valid_len + sample_offset : nullptr;
  a.B = B;
  a.Lv = Lv;
  a.npad = npad;
  a.sort = sort;
  a.add_prob = add_prob != 0;
  a.round_multiple = round_multiple;
  a.clip_length = clip_length;
  return launch_decode(a, stream, "univtg_decode_mr_pool");
}

extern "C" int univtg_temporal_nms(const double* windows, int32_t B, int32_t n, int32_t max_before_nms, double nms_thd,
                                   int32_t max_after_nms, double* out, int32_t* counts, void* stream) {
  using namespace uv;
  if (!windows || !out || !counts || B < 0 || n < 0 || max_before_nms < 0 || max_after_nms < 1) {
    set_error("univtg_temporal_nms: bad argument");
    return 1;
  }
  if (B == 0) return 0;
  const int n_in = n < max_before_nms ? n : max_before_nms;  // e["pred_relevant_windows"][:max_before_nms]
  if (n_in > 4096) {
    set_error("univtg_temporal_nms: more than 4096 candidates per sample");
    return 1;
  }
  NmsArgs a;
  memset(&a, 0, sizeof(a));
  a.windows = windows;
  a.out = out;
  a.counts = counts;
  a.thd = nms_thd;
  a.B = B;
  a.n = n;
  a.n_in = n_in;
  a.max_before = n_in;
  a.max_after = max_after_nms;
  return launch_nms(a, stream, "univtg_temporal_nms");
}

extern "C" int univtg_temporal_nms_pool(const double* rows, const int64_t* row_offsets, int32_t Q, int32_t max_rows,
                                        int32_t max_before_nms, double nms_thd, int32_t max_after_nms, int32_t sort, double* out,
                                        int32_t* counts, void* stream) {
  using namespace uv;
  if (!rows || !row_offsets || !out || !counts || Q < 0 || max_rows < 0 || max_before_nms < 0 || max_after_nms < 1) {
    set_error("univtg_temporal_nms_pool: bad argument");
    return 1;
  }
  if (Q == 0) return 0;
  const int n_in = max_rows < max_before_nms ? max_rows : max_before_nms;
  if (n_in > 4096) {
    set_error("univtg_temporal_nms_pool: more than 4096 candidates per query");
    return 1;
  }
  NmsArgs a;
  memset(&a, 0, sizeof(a));
  a.windows = rows;
  a.offsets = row_offsets;
  a.out = out;
  a.counts = counts;
  a.thd = nms_thd;
  a.B = Q;
  a.n = max_rows;
  a.n_in = n_in;
  a.max_before = max_before_nms;
  a.max_after = max_after_nms;
  a.sort = sort != 0;
  return launch_nms(a, stream, "univtg_temporal_nms_pool");
}
