// Shared between api.cu (forward orchestration) and train.cu (training workspace and backward): packed-weight layout,
// the buffers the forward writes, and the plan object behind the opaque univtg_plan handle.
#pragma once
#include <math.h>
#include <stdio.h>
#include <string.h>

#include "../../include/univtg_b200.h"
#include "backward.h"
#include "kernels.h"
#include "loss.h"
#include "ptx.cuh"
#include "rowops.h"

using namespace uv;

namespace {

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Host-side argument checks of the single-operator entry points: the message names the offending argument.
#define UV_REQ(cond, ...)      \
  do {                         \
    if (!(cond)) {             \
      set_error(__VA_ARGS__);  \
      return 1;                \
    }                          \
  } while (0)
inline bool al_(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) & (uintptr_t)(bytes - 1)) == 0; }
inline int pad64(int k) { return (k + 63) / 64 * 64; }

// ------------------------------------------------------------------------------------------------
// packed-weight layout
// ------------------------------------------------------------------------------------------------
struct ProjPacked {
  size_t ln_w, ln_b;  // fp32 [din]
  size_t w16;         // 16-bit [d, kpad]
  size_t bias;        // fp32 [d]  (last layer: linear bias + token-type embedding row)
  int din, kpad;
};
struct LayerPacked {
  size_t w_in;   // 16-bit [3d, d]  (rows: Wq, Wk, Wv)
  size_t b_in;   // fp32 [3d]
  size_t w_out;  // 16-bit [d, d]
  size_t b_out;
  size_t w1, b1;  // [ff, d], [ff]
  size_t w2, b2;  // [d, ff], [d]
  size_t n1w, n1b, n2w, n2b;
};
struct PackedLayout {
  ProjPacked vid[3], txt[3];
  LayerPacked layer[16];
  size_t conv1_w, conv1_b;                     // fused first conv of both heads: 16-bit [2d, 3d] (rows: class, span), fp32 [2d]
  size_t conv2c_w, conv2c_b, conv2s_w, conv2s_b;  // 16-bit [d, 3d], fp32 [d]
  size_t conv3c_w, conv3c_b, conv3s_w, conv3s_b;  // fp32 [3][d], [1], [2][3][d], [2]
  size_t pool_w;                                  // fp32 [d]
  size_t total;
};

// Order of the parameter tensors (univtg_pack_weights' params, univtg_backward's grads): per projector layer [ln.weight, ln.bias,
// W, b], video layers then text layers; token_type_embeddings; 12 tensors per encoder layer; span_embed.layers.{0,1,2} (weight,
// bias each), then class_embed's; weightedpool.weight.
struct ParamIndex {
  int np, nl;
  explicit ParamIndex(const univtg_config& c) : np(c.n_input_proj), nl(c.enc_layers) {}
  int vid(int i, int k) const { return 4 * i + k; }
  int txt(int i, int k) const { return 4 * np + 4 * i + k; }
  int type() const { return 8 * np; }
  int layer(int l, int k) const { return 8 * np + 1 + 12 * l + k; }
  int span(int k) const { return layer(nl, k); }
  int cls(int k) const { return span(6 + k); }
  int pool() const { return span(12); }
  int count() const { return pool() + 1; }
};

struct Cursor {
  size_t off = 0;
  size_t take(size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  }
};

bool check_cfg(const univtg_config* c) {
  if (!c) {
    set_error("null config");
    return false;
  }
  if (c->hidden_dim <= 0 || c->hidden_dim % 64 != 0) {
    set_error("hidden_dim %d must be a positive multiple of 64", c->hidden_dim);
    return false;
  }
  if (c->hidden_dim > 3072) {
    set_error("hidden_dim %d exceeds 3072, the widest LayerNorm that adds the residual branch in the same kernel", c->hidden_dim);
    return false;
  }
  if (c->nheads <= 0 || c->hidden_dim % c->nheads != 0) {
    set_error("nheads %d must divide hidden_dim %d", c->nheads, c->hidden_dim);
    return false;
  }
  if (c->dim_feedforward <= 0 || c->dim_feedforward % 64 != 0) {
    set_error("dim_feedforward %d must be a positive multiple of 64", c->dim_feedforward);
    return false;
  }
  if (c->enc_layers < 1 || c->enc_layers > 16) {
    set_error("enc_layers %d out of range [1,16]", c->enc_layers);
    return false;
  }
  if (c->n_input_proj < 1 || c->n_input_proj > 3) {
    set_error("n_input_proj %d out of range [1,3]", c->n_input_proj);
    return false;
  }
  if (c->v_feat_dim <= 0 || c->t_feat_dim <= 0) {
    set_error("feature dims must be positive");
    return false;
  }
  if (c->operand_format < 0 || c->operand_format > 2) {
    set_error("operand_format %d must be 0 (fp16), 1 (bf16) or 2 (fp16x3)", c->operand_format);
    return false;
  }
  return true;
}

// fp16x3 (operand_format 2) stores every 16-bit buffer as a hi plane (fp16) and a lo plane; the kernels then run with 16-bit
// format 0 and their split flag.  The lo planes of a buffer set (the packed weights, the inference workspace) form a second copy
// of that set's layout, placed right after it: the lo plane of a 16-bit buffer lies `total` bytes after its hi plane.
inline bool is_split(const univtg_config& c) { return c.operand_format == 2; }
inline int kernel_fmt(const univtg_config& c) { return is_split(c) ? 0 : c.operand_format; }
inline size_t planes(const univtg_config& c) { return is_split(c) ? 2 : 1; }
// Training keeps one 16-bit format per plan (gradients, AdamW repack); fp16x3 is an inference mode.
inline bool refuse_split(const univtg_config& c, const char* fn) {
  if (!is_split(c)) return false;
  set_error("%s: operand_format 2 (fp16x3) is an inference mode; training needs fp16 or bf16", fn);
  return true;
}
inline bool refuse_fmt2(int fmt, const char* fn) {
  if (fmt != 2) return false;
  set_error("%s: format 2 (fp16x3) is an inference mode; the backward operators take fp16 (0) or bf16 (1)", fn);
  return true;
}

PackedLayout make_layout(const univtg_config& c) {
  PackedLayout L;
  memset(&L, 0, sizeof(L));
  Cursor cur;
  const int d = c.hidden_dim, ff = c.dim_feedforward;
  for (int s = 0; s < 2; ++s) {
    ProjPacked* pp = s == 0 ? L.vid : L.txt;
    int din = s == 0 ? c.v_feat_dim : c.t_feat_dim;
    for (int i = 0; i < c.n_input_proj; ++i) {
      pp[i].din = din;
      pp[i].kpad = pad64(din);
      pp[i].ln_w = cur.take((size_t)din * 4);
      pp[i].ln_b = cur.take((size_t)din * 4);
      pp[i].w16 = cur.take((size_t)d * pp[i].kpad * 2);
      pp[i].bias = cur.take((size_t)d * 4);
      din = d;
    }
  }
  for (int l = 0; l < c.enc_layers; ++l) {
    LayerPacked& lp = L.layer[l];
    lp.w_in = cur.take((size_t)3 * d * d * 2);
    lp.b_in = cur.take((size_t)3 * d * 4);
    lp.w_out = cur.take((size_t)d * d * 2);
    lp.b_out = cur.take((size_t)d * 4);
    lp.w1 = cur.take((size_t)ff * d * 2);
    lp.b1 = cur.take((size_t)ff * 4);
    lp.w2 = cur.take((size_t)d * ff * 2);
    lp.b2 = cur.take((size_t)d * 4);
    lp.n1w = cur.take((size_t)d * 4);
    lp.n1b = cur.take((size_t)d * 4);
    lp.n2w = cur.take((size_t)d * 4);
    lp.n2b = cur.take((size_t)d * 4);
  }
  L.conv1_w = cur.take((size_t)2 * d * 3 * d * 2);
  L.conv1_b = cur.take((size_t)2 * d * 4);
  L.conv2c_w = cur.take((size_t)d * 3 * d * 2);
  L.conv2c_b = cur.take((size_t)d * 4);
  L.conv2s_w = cur.take((size_t)d * 3 * d * 2);
  L.conv2s_b = cur.take((size_t)d * 4);
  L.conv3c_w = cur.take((size_t)3 * d * 4);
  L.conv3c_b = cur.take(4);
  L.conv3s_w = cur.take((size_t)2 * 3 * d * 4);
  L.conv3s_b = cur.take(8);
  L.pool_w = cur.take((size_t)d * 4);
  L.total = cur.off;
  return L;
}

// ------------------------------------------------------------------------------------------------
// pack kernels
// ------------------------------------------------------------------------------------------------
// All (re)packing work of one univtg_pack_weights call is described by a task table and executed by a handful of launches
// (the table travels as a kernel parameter, <= 4 KB per launch) instead of ~75 tiny kernels.
struct PackTask {
  const float* src;
  const float* add;  // kind 3: optional second vector added element-wise
  void* dst;
  int kind;          // 0: rows -> 16-bit [rows, ld] zero-padded, 1: conv [N,C,3] -> 16-bit [N, 3C], 2: conv -> fp32 [N,3,C], 3: vector copy(+add)
  int rows, cols, ld;
  int blk0;          // first block of this task in the launch (blocks are dealt out in proportion to the task's size)
};
constexpr int kPackTasksPerLaunch = 64;
constexpr int kPackItemsPerBlock = 256 * 8;  // work items per block (an item = 4 output elements, or one conv (n, c) pair)
struct PackTable {
  int n, fmt;
  long long lo;  // fp16x3: bytes from a 16-bit destination to its lo plane (0: one plane)
  PackTask t[kPackTasksPerLaunch];
};

inline size_t pack_task_items(const PackTask& k) {
  if (k.kind == 0) return ((size_t)k.rows * k.ld + 3) / 4;  // ld % 4 == 0 for every packed matrix (K padded to 64)
  if (k.kind == 1 || k.kind == 2) return (size_t)k.rows * k.cols;
  return ((size_t)k.rows + 3) / 4;
}

template <bool SPLIT = false>  // SPLIT: fp16x3, the 16-bit kinds also write their lo planes (tab.lo)
__global__ void __launch_bounds__(256) pack_multi_kernel(const __grid_constant__ PackTable tab) {
  pdl_prologue();
  int ti = 0;
  while (ti + 1 < tab.n && (int)blockIdx.x >= tab.t[ti + 1].blk0) ++ti;
  const PackTask& k = tab.t[ti];
  const int fmt = tab.fmt;
  const size_t first = (size_t)(blockIdx.x - k.blk0) * kPackItemsPerBlock;
  if (k.kind == 0) {
    const size_t items = ((size_t)k.rows * k.ld) / 4;
    const bool dense = k.ld == k.cols && (k.cols & 3) == 0 && (((uintptr_t)k.src) & 15) == 0;
    uint2* dst2 = reinterpret_cast<uint2*>(k.dst);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const size_t it = first + u * 256 + threadIdx.x;
      if (it >= items) break;
      float4 v;
      if (dense) {
        v = __ldg(reinterpret_cast<const float4*>(k.src) + it);
      } else {
        const int r = (int)((it * 4) / k.ld), c = (int)((it * 4) % k.ld);  // 4 consecutive columns of one row (ld % 4 == 0)
        const float* row = k.src + (size_t)r * k.cols;
        v.x = c + 0 < k.cols ? __ldg(row + c + 0) : 0.f;
        v.y = c + 1 < k.cols ? __ldg(row + c + 1) : 0.f;
        v.z = c + 2 < k.cols ? __ldg(row + c + 2) : 0.f;
        v.w = c + 3 < k.cols ? __ldg(row + c + 3) : 0.f;
      }
      dst2[it] = make_uint2(cvt16x2(v.x, v.y, fmt), cvt16x2(v.z, v.w, fmt));
      if constexpr (SPLIT) reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(k.dst) + tab.lo)[it] = make_uint2(cvt16x2_lo(v.x, v.y), cvt16x2_lo(v.z, v.w));
    }
  } else if (k.kind == 1 || k.kind == 2) {
    // item = one (n, c) pair: three consecutive source floats (taps), scattered to the three tap planes of row n
    const int C = k.cols;
    const size_t items = (size_t)k.rows * C;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const size_t it = first + u * 256 + threadIdx.x;
      if (it >= items) break;
      const int n = (int)(it / C), c = (int)(it % C);
      const float* sp = k.src + it * 3;
      const float v0 = __ldg(sp), v1 = __ldg(sp + 1), v2 = __ldg(sp + 2);
      const size_t o = (size_t)n * 3 * C + c;
      if (k.kind == 1) {
        uint16_t* d16 = reinterpret_cast<uint16_t*>(k.dst);
        d16[o] = cvt16(v0, fmt);
        d16[o + C] = cvt16(v1, fmt);
        d16[o + 2 * C] = cvt16(v2, fmt);
        if constexpr (SPLIT) {
          uint16_t* l16 = reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(k.dst) + tab.lo);
          l16[o] = cvt16_lo(v0);
          l16[o + C] = cvt16_lo(v1);
          l16[o + 2 * C] = cvt16_lo(v2);
        }
      } else {
        float* d32 = reinterpret_cast<float*>(k.dst);
        d32[o] = v0;
        d32[o + C] = v1;
        d32[o + 2 * C] = v2;
      }
    }
  } else {
    float* dst = reinterpret_cast<float*>(k.dst);
    for (int u = 0; u < 8 * 4; ++u) {
      const size_t i = first * 4 + (size_t)u * 256 + threadIdx.x;
      if (i >= (size_t)k.rows) break;
      dst[i] = k.src[i] + (k.add ? k.add[i] : 0.f);
    }
  }
}

struct Packer {
  uint8_t* base;
  int fmt;
  long long lo;  // fp16x3: bytes to the lo planes
  cudaStream_t st;
  PackTable tab;
  bool skip_matrices = false;  // only the fp32 vectors / small tensors (kinds 2, 3)
  void push(const PackTask& t) {
    if (skip_matrices && (t.kind == 0 || t.kind == 1)) return;
    if (tab.n == kPackTasksPerLaunch) flush();
    tab.t[tab.n++] = t;
  }
  void flush() {
    if (tab.n == 0) return;
    tab.fmt = fmt;
    tab.lo = lo;
    int blocks = 0;
    for (int i = 0; i < tab.n; ++i) {
      tab.t[i].blk0 = blocks;
      blocks += (int)((pack_task_items(tab.t[i]) + kPackItemsPerBlock - 1) / kPackItemsPerBlock);
    }
    if (blocks > 0) {
      if (lo) launch_k(pack_multi_kernel<true>, dim3(blocks), dim3(256), 0, st, tab);
      else launch_k(pack_multi_kernel<false>, dim3(blocks), dim3(256), 0, st, tab);
    }
    tab.n = 0;
  }
  void rows(const float* src, size_t off, int rows_, int cols, int ld) { push(PackTask{src, nullptr, base + off, 0, rows_, cols, ld, 0}); }
  void conv(const float* src, size_t off, int N, int C) { push(PackTask{src, nullptr, base + off, 1, N, C, 0, 0}); }
  void conv_f32(const float* src, size_t off, int N, int C) { push(PackTask{src, nullptr, base + off, 2, N, C, 0, 0}); }
  void vec(const float* src, size_t off, int n, const float* add = nullptr) { push(PackTask{src, add, base + off, 3, n, 0, 0, 0}); }
};

}  // namespace

// ------------------------------------------------------------------------------------------------
// buffers the forward writes
// ------------------------------------------------------------------------------------------------
// Training keeps one buffer per layer and the statistics the backward needs (TrainWs, train.cu).  Inference
// (make_infer_ws) lets every per-layer entry alias one buffer and leaves the training-only entries null.
struct FwdBufs {
  uint16_t *a_vid[3], *a_txt[3];   // LN'd 16-bit projector inputs
  float *pmean_v[3], *prstd_v[3], *pmean_t[3], *prstd_t[3];  // projector LayerNorm statistics (training)
  float *p_vid32[3], *p_txt32[3];  // output of projector layer i (input of LayerNorm i+1)
  float* txtproj32;                // [Mt, d] projected text tokens (+type embedding)
  float* pool_alpha;               // [B, Lt] pooling softmax weights (training)
  float *pos, *key_mask, *pool_logits;
  float* dp_scale;                 // [2 * enc_layers, B] DropPath scales drawn in-kernel (training; reused by the backward)
  uint16_t *xin16[17], *xpos16[17];  // operands of layer l's in-projections (index enc_layers: output of the last layer)
  uint16_t *qkv16[16], *attn16[16], *x1_16[16], *h16[16];
  float *lse[16], *y1[16], *mean1[16], *rstd1[16], *y2[16], *mean2[16], *rstd2[16];  // training
  uint16_t* dgelu16[16];           // GELU'(pre-activation) of the FFN, written by FFN1's epilogue beside h16 (training)
  float *x32, *x1_32;              // fp32 residual stream before / after LayerNorm 1 (the same buffer in inference)
  uint16_t *hA, *h1, *hc2, *hs2;   // conv-head buffers (separated layout)
  uint16_t* br16;                  // DropPath-scaled residual branch (out-proj / FFN2 output)
  float *pred_logits, *pred_spans;  // copies of the outputs the backward needs (training)
  size_t total;
};

// ------------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------------
constexpr int kMaxMarks = 640;
struct univtg_plan {
  univtg_config cfg;
  univtg_shape shp;
  PackedLayout lay;
  const uint8_t* packed;
  uint8_t* ws;
  const float* dim_t;
  int num_sms;
  int in_fmt;       // src_vid / src_txt element type: 0 f32 (reference collate), 1 fp16, 2 bf16 (packed feature shards)
  int num_sms_bwd;  // SM budget of the backward's GEMM launches (0: num_sms); see univtg_plan_set_backward_sm_budget
  float attn_dropout;  // p of the attention dropout of univtg_forward_train / univtg_backward (0: off); univtg_forward ignores it
  // device seed of the train-mode randomness (univtg_plan_set_seed_source; null: rng->seed).  Kernels read it at their start, so a
  // CUDA graph captured with it set draws the masks of whatever seed univtg_rng_advance wrote ahead of each replay.
  const unsigned long long* seed_dev = nullptr;
  int txt_pos_on;           // learned text positions (univtg_plan_set_txt_pos); 0: off
  long long pk_lo, ws_lo;   // fp16x3: elements from a 16-bit weight / workspace buffer to its lo plane (0: one plane)
  univtg_txt_pos txt_pos;
  int B, Lv, Lt, L, d, ff, H, dh, M, Mv, Mt, Mh;
  int bn_proj[3];  // tile widths of the forward's GEMM launches (tile_for)
  int bn_qkv, bn_out, bn_ffn1, bn_ffn2, bn_conv1, bn_conv2;
  int launches;
  // optional "gradients of stage k are final" events recorded by univtg_backward (gradient-exchange overlap)
  int n_grad_events;
  cudaEvent_t grad_events[24];
  // optional per-launch CUDA-event timeline (bench / profiling only)
  int profiling;
  int n_marks;
  cudaEvent_t marks[kMaxMarks];
  int mark_kind[kMaxMarks];  // kind of the interval that ENDS at mark i (i >= 1): 0 row kernel, 1 tensor-core GEMM, 2 attention, 3 other work
};

namespace {
// dropout spec of the forward / backward of plan P: rng->seed, or the plan's device seed when one is set
inline uv::DropSpec plan_drop_spec(const univtg_plan* P, const univtg_rng* rng, unsigned int stream, float p) {
  uv::DropSpec s = uv::make_drop_spec(rng->seed, stream, p);
  s.seed_ptr = P->seed_dev;
  return s;
}

inline void prof_begin(univtg_plan* P, cudaStream_t st) {
  if (!P->profiling) return;
  P->n_marks = 0;
  if (!P->marks[0]) cudaEventCreate(&P->marks[0]);
  cudaEventRecord(P->marks[0], st);
  P->mark_kind[0] = -1;
  P->n_marks = 1;
}
inline void prof_mark(univtg_plan* P, cudaStream_t st, int kind) {
  if (!P->profiling || P->n_marks >= kMaxMarks) return;
  const int i = P->n_marks;
  if (!P->marks[i]) cudaEventCreate(&P->marks[i]);
  cudaEventRecord(P->marks[i], st);
  P->mark_kind[i] = kind;
  P->n_marks = i + 1;
}
// The forward records a mark after every launch.  The backward brackets each GEMM / attention launch by two marks, so that the
// interval ending at the second mark is that kernel alone (the interval ending at the first one - kind 3 - collects whatever ran
// since the previous mark).
inline int gemm_launch(univtg_plan* P, GemmGroup& g, int bn, int sms, cudaStream_t st) {
  prof_mark(P, st, 3);
  const int rc = launch_gemm_group(g, bn, sms, st);
  prof_mark(P, st, 1);
  return rc;
}

// Empties `g` for `num` problems in 16-bit format `fmt`; split / lo16: fp16x3 (GemmGroup).
inline void reset_group(GemmGroup& g, int num, int fmt, int split = 0, long long lo16 = 0) {
  memset(&g, 0, sizeof(g));
  g.num = num;
  g.fmt = fmt;
  g.split = split;
  g.lo16 = lo16;
}

// Longest sequence the SIMT attention backward can stage (attention_bwd_simt_smem = 32 L bytes) in the device's opt-in shared
// memory per block.  Without a device to ask, the sm_90 value (227 KB, the only target the library is built for) is used.
inline int attention_bwd_simt_max_L() {
  int dev = 0, optin = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
      optin <= 0) {
    cudaGetLastError();
    optin = 227 * 1024;
  }
  return (int)((size_t)optin / attention_bwd_simt_smem(1));
}

// Arguments of the attention core backward over qkv [B*L, 3d] and dO [B*L, d], both in 16-bit format `fmt` (d = H dh), for
// attention_bwd_route; the caller adds the dropout spec.
inline AttnBwdArgs attention_bwd_args(const void* qkv, const void* dO, const float* key_mask, const float* lse, const float* delta,
                                      float* dqkv32, int B, int L, int H, int dh, int fmt) {
  AttnBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.qkv = reinterpret_cast<const uint16_t*>(qkv);
  a.dO = reinterpret_cast<const uint16_t*>(dO);
  a.key_mask = key_mask;
  a.lse = lse;
  a.delta = delta;
  a.dqkv32 = dqkv32;
  a.scale = 1.0f / sqrtf((float)dh);
  a.B = B;
  a.L = L;
  a.H = H;
  a.dh = dh;
  a.d = H * dh;
  a.fmt_act = a.fmt_grad = fmt;
  return a;
}

// Routing of the attention core backward, shared by univtg_backward and the single-operator entry points.  `a` holds everything but
// dq_atomic, dqkv16 and the tensor maps.  tc: wgmma kernel (dh 64 / 128), else the SIMT kernel.  dQ | dK | dV go
//   dq_mode 0: straight to the 16-bit operand dqkv16 (tc, one key tile L <= 128, dqkv16 given); dqkv32 is not written,
//   dq_mode 1: to dqkv32, dQ stored (tc, one key tile, no dqkv16),
//   dq_mode 2: to dqkv32 after a memset, dQ accumulated atomically (several key tiles, or SIMT).
// P (optional): the plan whose profiling marks bracket the wgmma launch.
inline int attention_bwd_route(AttnBwdArgs& a, bool tc, uint16_t* dqkv16, cudaStream_t st, int* dq_mode, int* kernel_used = nullptr,
                               univtg_plan* P = nullptr) {
  const int M = a.B * a.L, d = a.d;
  a.dq_atomic = (!tc || a.L > 128) ? 1 : 0;
  a.dqkv16 = a.dq_atomic ? nullptr : dqkv16;
  if (dq_mode) *dq_mode = a.dq_atomic ? 2 : (a.dqkv16 ? 0 : 1);
  if (a.dq_atomic) cudaMemsetAsync(a.dqkv32, 0, (size_t)M * 3 * d * 4, st);
  if (!tc) return launch_attention_bwd_simt(a, st, kernel_used);
  if (make_tmap_2d(&a.tm_qkv, a.qkv, (uint64_t)M, (uint64_t)3 * d, (uint64_t)3 * d, 128, 64)) return 1;
  if (make_tmap_2d(&a.tm_do, a.dO, (uint64_t)M, (uint64_t)d, (uint64_t)d, 128, 64)) return 1;
  if (P) prof_mark(P, st, 3);
  const int rc = launch_attention_bwd(a, st, kernel_used);
  if (P) prof_mark(P, st, 2);
  return rc;
}
}  // namespace

namespace {

void init_problem(GemmProblem& p) {
  memset(&p, 0, sizeof(p));
  p.taps = 1;
  p.ksplit = 1;
  p.alpha = 1.f;
  p.a_fmt = p.b_fmt = p.out_fmt = -1;
  p.colsum_scale = 1.f;
  // default coordinate rules: K-major A [M,K] and B [N,K]
  p.ca = OperandCoord{0, 0, 0, 1, 0, 1, 0, 0};
  p.cb = OperandCoord{0, 0, 0, 1, 0, 1, 0, 0};
}

struct Mat16 {  // row-major 16-bit matrix view
  const uint16_t* p;
  int rows, cols, ld;
};

// Operand map of a K-major 16-bit matrix: a plain 2-D map, or with lo > 0 (fp16x3) a hi / lo pair `lo` elements apart.
inline int make_tmap_op(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t box_cols,
                        long long lo) {
  return lo ? make_tmap_split(m, base, rows, cols, ld, box_rows, box_cols, (uint64_t)lo) : make_tmap_2d(m, base, rows, cols, ld, box_rows, box_cols);
}

// C[M,N] = sum_k A(m,k) B(n,k).  a_mn: A is stored [K rows, M cols] (else [M rows, K cols]); same for B.
// lo_a / lo_b > 0: fp16x3 operands (K-major only) whose lo planes lie that many elements after A / B.
int setup_gemm(GemmProblem& p, Mat16 A, int a_mn, Mat16 B, int b_mn, int M, int N, int K, int bn, long long lo_a = 0,
               long long lo_b = 0) {
  init_problem(p);
  if ((lo_a || lo_b) && (a_mn || b_mn || !lo_a || !lo_b)) {
    set_error("fp16x3 GEMM operands must both be split and K-major");
    return 1;
  }
  p.M = M;
  p.N = N;
  p.a_mn = a_mn;
  p.b_mn = b_mn;
  p.kblk_per_tap = (K + 63) / 64;
  int rc = 0;
  if (!a_mn) {
    rc |= make_tmap_op(&p.tm_a, A.p, (uint64_t)A.rows, (uint64_t)A.cols, (uint64_t)A.ld, GEMM_BM, 64, lo_a);
  } else {
    rc |= make_tmap_2d(&p.tm_a, A.p, (uint64_t)A.rows, (uint64_t)A.cols, (uint64_t)A.ld, 64, 64);
    p.ca = OperandCoord{0, 1, 0, 0, 0, 0, 0, 1};
  }
  if (!b_mn) {
    rc |= make_tmap_op(&p.tm_b, B.p, (uint64_t)B.rows, (uint64_t)B.cols, (uint64_t)B.ld, (uint32_t)bn, 64, lo_b);
    p.b_box_rows = bn;
  } else {
    rc |= make_tmap_b_mn(p, B.p, (uint64_t)B.rows, (uint64_t)B.cols, (uint64_t)B.ld, bn);
    p.cb = OperandCoord{0, 1, 0, 0, 0, 0, 0, 1};
  }
  return rc;
}

// k=3 Conv1d (padding 1) forward in the conv-head layout (buffer row = logical row + 1; rows 0 and Mh + 1 and every sample's
// separator row of X are zeros): Y[m] = sum_t X[m + t - 1] W[:, :, t] over Mh logical rows.  A = X [Mh + 2, Cin] (pitch lda,
// K-major, row-shifted by the tap), B = packed W [N, 3 Cin] (K-major, w2[o, t * Cin + c] = W[o, c, t]); K = 3 taps x Cin
// (Cin % 64 == 0).  lo_a / lo_b > 0: fp16x3 operands whose lo planes lie that many elements after X / W.
int conv_fwd_problem(GemmProblem& p, int Mh, const uint16_t* X, int lda, int Cin, const uint16_t* Wp, int N, int bn, long long lo_a = 0,
                     long long lo_b = 0) {
  init_problem(p);
  p.M = Mh;
  p.N = N;
  p.taps = 3;
  p.kblk_per_tap = Cin / 64;
  p.ca = OperandCoord{0, 0, 0, 1, 0, 1, 1, 0};    // rows m0 + t (buffer row of logical row m0 + t - 1), cols k
  p.cb = OperandCoord{0, 0, Cin, 1, 0, 1, 0, 0};  // cols t * Cin + k, rows n0
  int r = make_tmap_op(&p.tm_a, X, (uint64_t)Mh + 2, (uint64_t)Cin, (uint64_t)lda, GEMM_BM, 64, lo_a);
  r |= make_tmap_op(&p.tm_b, Wp, (uint64_t)N, (uint64_t)3 * Cin, (uint64_t)3 * Cin, (uint32_t)bn, 64, lo_b);
  p.b_box_rows = bn;
  return r;
}

// k=3 Conv1d backward in the conv-head layout (buffer row = logical row + 1; rows 0, Mh + 1 and every sample's separator row are
// zeros).
// dgrad: dX[m] = sum_t' dY[m + t' - 1] W[:, :, 2 - t'] over Mh logical rows.  A = dY [Mh + 2, Kc] (pitch ldy, K-major, row-shifted
// by the tap), B = packed W [Kc, 3 * Cin] (MN-major, w2[o, t * Cin + c] = W[o, c, t]); N = Cin, K = 3 taps x Kc (Kc % 64 == 0).
int conv_dgrad_problem(GemmProblem& p, int Mh, const uint16_t* dY, int ldy, int Kc, const uint16_t* Wp, int Cin, int bn) {
  init_problem(p);
  p.M = Mh;
  p.N = Cin;
  p.taps = 3;
  p.kblk_per_tap = Kc / 64;
  p.b_mn = 1;
  p.ca = OperandCoord{0, 0, 0, 1, 0, 1, 1, 0};           // rows m0 + t', cols k
  p.cb = OperandCoord{2 * Cin, 1, -Cin, 0, 0, 0, 0, 1};  // cols n0 + (2 - t') * Cin, rows k (out channel)
  int r = make_tmap_2d(&p.tm_a, dY, (uint64_t)Mh + 2, (uint64_t)Kc, (uint64_t)ldy, GEMM_BM, 64);
  r |= make_tmap_b_mn(p, Wp, (uint64_t)Kc, (uint64_t)3 * Cin, (uint64_t)3 * Cin, bn);
  return r;
}
// wgrad of tap t: dW[n, c, t] = sum_m dY[m, n] X[m + t - 1, c] over Mh logical rows.  A = dY [Mh + 2, Nc] (pitch ldy, MN-major),
// B = X [Mh + 2, Cin] (pitch ldx, MN-major, row-shifted by t); M = Nc, N = Cin, K = Mh.
int conv_wgrad_problem(GemmProblem& p, int Mh, const uint16_t* dY, int ldy, int Nc, const uint16_t* X, int ldx, int Cin, int t, int bn) {
  init_problem(p);
  p.M = Nc;
  p.N = Cin;
  p.a_mn = 1;
  p.b_mn = 1;
  p.kblk_per_tap = (Mh + 63) / 64;
  p.ca = OperandCoord{0, 1, 0, 0, 1, 0, 0, 1};  // cols m0 (out channel), rows 1 + k
  p.cb = OperandCoord{0, 1, 0, 0, t, 0, 0, 1};  // cols n0 (in channel), rows t + k
  int r = make_tmap_2d(&p.tm_a, dY, (uint64_t)Mh + 2, (uint64_t)Nc, (uint64_t)ldy, 64, 64);
  r |= make_tmap_b_mn(p, X, (uint64_t)Mh + 2, (uint64_t)Cin, (uint64_t)ldx, bn);
  return r;
}

// K-major linear problem: A [M, K] (pitch lda), W [N, K] (pitch ldw).
inline int setup_linear(GemmProblem& p, const uint16_t* A, int M, int K, int lda, const uint16_t* W, int N, int ldw, int bn,
                        long long lo_a = 0, long long lo_w = 0) {
  return setup_gemm(p, Mat16{A, M, K, lda}, 0, Mat16{W, N, K, ldw}, 0, M, N, K, bn, lo_a, lo_w);
}

// Tile width + split-K factors for one grouped launch (cost model: choose_tile, gemm.cu).  K in elements; step 16 when every B
// operand is K-major, 64 when one is MN-major; split: split-K limit of the problem (1, the default, for a problem whose epilogue
// cannot accumulate).
struct MNK {
  int M, N, K;
  int split = 1;
};
inline TileChoice tile_for(int sms, int step, MNK a, MNK b = MNK{0, 0, 0}, MNK c3 = MNK{0, 0, 0}, MNK c4 = MNK{0, 0, 0}) {
  const MNK all[GEMM_MAX_GROUP] = {a, b, c3, c4};
  int Ms[GEMM_MAX_GROUP], Ns[GEMM_MAX_GROUP], kb[GEMM_MAX_GROUP], ms[GEMM_MAX_GROUP], num = 0;
  for (const MNK& x : all) {
    if (x.M <= 0) break;
    Ms[num] = x.M;
    Ns[num] = x.N;
    kb[num] = (x.K + 63) / 64;
    ms[num] = x.split;
    ++num;
  }
  return choose_tile(Ms, Ns, kb, ms, num, sms, step);
}

// Inference workspace: one buffer per role, shared by all layers; LayerNorm 1 works in place on the residual stream.
FwdBufs make_infer_ws(const univtg_config& c, const univtg_shape& s, const PackedLayout& L, uint8_t* base) {
  FwdBufs w;
  memset(&w, 0, sizeof(w));
  Cursor cur;
  const size_t d = c.hidden_dim, ff = c.dim_feedforward;
  const size_t B = s.batch, Lv = s.l_vid, Lt = s.l_txt, Lc = Lv + Lt;
  const size_t M = B * Lc, Mv = B * Lv, Mt = B * Lt, Mh = B * (Lv + 1);
  auto take16 = [&](size_t elems) { return reinterpret_cast<uint16_t*>(base + cur.take(elems * 2)); };
  auto take32 = [&](size_t elems) { return reinterpret_cast<float*>(base + cur.take(elems * 4)); };
  for (int i = 0; i < c.n_input_proj; ++i) {
    w.a_vid[i] = take16(Mv * L.vid[i].kpad);
    w.a_txt[i] = take16(Mt * L.txt[i].kpad);
  }
  float* p_vid32 = take32(Mv * d);
  float* p_txt32 = take32(Mt * d);
  w.txtproj32 = take32(Mt * d);
  w.pos = take32(Mv * d);
  w.key_mask = take32(B * Lc);
  w.pool_logits = take32(B * Lt);
  w.x32 = w.x1_32 = take32(M * d);
  w.br16 = take16(M * d);
  uint16_t* x16 = take16(M * d);
  uint16_t* xpos16 = take16(M * d);
  uint16_t* qkv16 = take16(M * 3 * d);
  uint16_t* attn16 = take16(M * d);
  uint16_t* h16 = take16(M * ff);
  w.hA = take16((Mh + 2) * d);
  w.h1 = take16((Mh + 2) * 2 * d);
  w.hc2 = take16((Mh + 2) * d);
  w.hs2 = take16((Mh + 2) * d);
  w.total = cur.off;
  for (int i = 0; i < c.n_input_proj; ++i) {
    w.p_vid32[i] = p_vid32;
    w.p_txt32[i] = p_txt32;
  }
  for (int l = 0; l <= c.enc_layers; ++l) {
    w.xin16[l] = x16;
    w.xpos16[l] = xpos16;
  }
  for (int l = 0; l < c.enc_layers; ++l) {
    w.qkv16[l] = qkv16;
    w.attn16[l] = attn16;
    w.x1_16[l] = x16;
    w.h16[l] = h16;
  }
  return w;
}

// Scratch of the learned text positions (univtg_txt_pos.scratch, univtg_txt_pos_scratch_bytes): pos_t for the encoder layers'
// q/k operands; training adds its LayerNorm statistics and the backward's accumulators.
struct TxtPosWs {
  float* pos;       // [Mt, d] pos_t
  float *mean, *rstd;  // [Mt] (training)
  float* dpos;      // [Mt, d] gradient of pos_t summed over the encoder layers (training)
  uint16_t* dqk16;  // [Mt, 2d] text rows of [dq | dk] of the layer being differentiated (training)
  size_t total;
};
inline TxtPosWs make_txt_pos_ws(const univtg_config& c, const univtg_shape& s, void* base_) {
  TxtPosWs w;
  memset(&w, 0, sizeof(w));
  uint8_t* base = reinterpret_cast<uint8_t*>(base_);
  Cursor cur;
  const size_t d = c.hidden_dim, Mt = (size_t)s.batch * s.l_txt;
  w.pos = reinterpret_cast<float*>(base + cur.take(Mt * d * 4));
  if (s.training) {
    w.mean = reinterpret_cast<float*>(base + cur.take(Mt * 4));
    w.rstd = reinterpret_cast<float*>(base + cur.take(Mt * 4));
    w.dpos = reinterpret_cast<float*>(base + cur.take(Mt * d * 4));
    w.dqk16 = reinterpret_cast<uint16_t*>(base + cur.take(Mt * 2 * d * 2));
  }
  w.total = cur.off;
  return w;
}

bool check_shape(const univtg_shape* s) {
  if (!s || s->batch < 1 || s->l_vid < 1 || s->l_txt < 1) {
    set_error("bad shape");
    return false;
  }
  return true;
}

}  // namespace

// Reference Model.forward (model/univtg.py:105-155) over the buffers `W`, for univtg_forward and univtg_forward_train (api.cu).
// drop_masks / rng: train-mode randomness as univtg_forward_train takes it (NULL at inference; attention dropout applies only with
// an rng, P->attn_dropout > 0).  The training-only entries of `W` that are non-null are written as well.
int run_forward(univtg_plan* P, const FwdBufs& W, const float* src_txt, const float* src_txt_mask, const float* src_vid,
                const float* src_vid_mask, const float* droppath_scale, const float* const* drop_masks, const univtg_rng* rng,
                float* pred_logits, float* pred_spans, float* vid_mem_proj, float* txt_mem_proj, float* saliency_scores,
                cudaStream_t st);

