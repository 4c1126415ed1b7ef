// Launchers of the backward-pass kernels (backward.cu, attention_bwd.cu).  SURVEY.md A.6 lists the math.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "philox.cuh"

namespace uv {

// LayerNorm backward over rows:  xhat = (y - mean) * rstd,  g = dout * gamma,
//   dy = rstd * (g - mean_j(g) - xhat * mean_j(g * xhat));  dgamma += sum_rows dout * xhat;  dbeta += sum_rows dout
struct LnBwdArgs {
  const float* dout;  // [rows, ld_dout] gradient w.r.t. the LayerNorm output
  int ld_dout;
  const float* y;     // [rows, ld_y] LayerNorm input saved by the forward pass
  int ld_y;
  const uint16_t* y16;  // alternative: the LayerNorm input as 16-bit (first projector layer fed from a 16-bit feature shard)
  int y_fmt;
  const float* mean;  // [rows]
  const float* rstd;  // [rows]
  const float* gamma; // [d]
  int rows, d;
  const float* row_scale;  // per-sample DropPath scale (indexed by row / L) applied to the 16-bit branch gradient, or null
  int L;
  int relu_mask_y;         // 1: the LayerNorm input is a ReLU output; gradient is zeroed where y <= 0 (projector chain)
  float* dy32;             // [rows, d] fp32 dy (residual-stream gradient) or null
  uint16_t* dbr16;         // [rows, ld16] 16-bit (row_scale * dy [masked]) = gradient of the producing branch, or null
  int ld16;
  int fmt16;
  float* dgamma;           // [d] atomically accumulated, or null
  float* dbeta;            // [d]
  float* colsum;           // [d] atomically accumulated column sums of the values written to dbr16 (bias gradient), or null
  float pgrad_scale;       // factor on dgamma / dbeta / colsum (1 / loss-scale: parameter gradients leave unscaled)
  const float* dout_mul;   // optional [rows, d] multiplier applied to dout on load (input-dropout mask incl. 1/(1-p))
  DropSpec drop;           // in-kernel regeneration of the forward's input-dropout multipliers (drop.on; ignored with dout_mul)
};
// kernel_used (optional): which instantiation ran (LnbKernel; the same numbering as univtg_op_layernorm_bwd reports)
enum LnbKernel { LNB_PARAMS = 0, LNB_WARP2 = 1, LNB_WARP4 = 2, LNB_WARP8 = 3, LNB_VEC1 = 4, LNB_VEC2 = 5, LNB_ROW8 = 6, LNB_ROW24 = 7 };
int launch_layernorm_bwd(const LnBwdArgs& a, cudaStream_t stream, int* kernel_used = nullptr);

// Optional compact copy of the text rows (row r = b*L + l, l >= Lv) of the first txt_cols columns of the 16-bit output, as
// [B*(L-Lv), txt_cols] (the [dq | dk] rows the learned text positions' gradient needs); txt16 == NULL: no copy.
struct TxtRows {
  uint16_t* txt16;
  int L, Lv, txt_cols;
};

// out16[r, c] = cvt(in32[r, c]) (+ column sums), rows x cols with leading dims
int launch_cvt16_colsum(const float* in32, int ld_in, uint16_t* out16, int ld_out, int rows, int cols, int fmt, float* colsum,
                        float colsum_scale, cudaStream_t stream, TxtRows txt = TxtRows{nullptr, 0, 0, 0});

// dst[n][c][t] = src[t][n][c], t < 3 (conv weight gradient planes -> reference [out, in, 3] layout)
int launch_tap_interleave(const float* src, float* dst, int N, int C, cudaStream_t stream);

// colsum[c] += scale * sum_r in16[r, c]
int launch_colsum16(const uint16_t* in16, int ld, int rows, int cols, int fmt, float* colsum, float scale, cudaStream_t stream,
                    TxtRows txt = TxtRows{nullptr, 0, 0, 0});

// delta[b, h, i] = sum_c dO[b, i, h, c] * O[b, i, h, c].  vec_used (optional): 1 when the 128-bit vector path ran, 0 scalar.
int launch_attn_delta(const uint16_t* dO, int fmt_do, const uint16_t* O, int fmt_o, float* delta, int B, int L, int H, int dh,
                      cudaStream_t stream, int* vec_used = nullptr);

struct AttnBwdArgs {
  CUtensorMap tm_qkv;  // [B*L, 3d] 16-bit activations (Q | K | V), box {64, 128}
  CUtensorMap tm_do;   // [B*L, d] 16-bit gradient of the attention output, box {64, 128}
  const uint16_t* qkv; // same buffers through plain pointers (SIMT path)
  const uint16_t* dO;
  const float* key_mask;  // [B, L]
  const float* lse;       // [B, H, L]
  const float* delta;     // [B, H, L]
  float* dqkv32;          // [B*L, 3d] fp32: dQ (accumulated atomically over key tiles) | dK | dV
  float scale;
  int B, L, H, dh, d;
  int fmt_act, fmt_grad;  // formats of qkv / dO
  int dq_atomic;          // 1 when dqkv32 was pre-zeroed and dQ must be accumulated (more than one key tile or SIMT path)
  // Single-key-tile fast path (L <= 128, tensor-core kernel): write dQ | dK | dV directly as 16-bit operands of the in-projection
  // dgrad / wgrad GEMMs; dqkv32 is then not written (the in_proj_bias gradient comes from launch_colsum16 over this buffer).
  uint16_t* dqkv16;       // [B*L, 3d] or null
  DropSpec drop;          // the forward's attention dropout (drop.on): dV += (P o M)^T dO, dS = P o (M o dP - delta)
};
// kernel_used (optional): which instantiation ran, the numbering univtg_op_attention_bwd_full reports:
// wgmma 4 (dh 128) + 2 (bf16) + dropout = 0..7, SIMT 8 + dropout.
int launch_attention_bwd(const AttnBwdArgs& a, cudaStream_t stream, int* kernel_used = nullptr);       // wgmma, dh in {64, 128}
int launch_attention_bwd_simt(const AttnBwdArgs& a, cudaStream_t stream, int* kernel_used = nullptr);  // any dh; dqkv32 pre-zeroed
// Dynamic shared memory of the SIMT kernel: p and dS of L keys for each of its 4 warps.
inline size_t attention_bwd_simt_smem(int L) { return (size_t)4 * 2 * L * sizeof(float); }

// ---- conv heads: last layer (1 / 2 output channels) ----
struct HeadFinalBwdArgs {
  const float* g_logits;     // [B, Lv] dL/d pred_logits
  const float* g_spans;      // [B, Lv, 2]
  const float* pred_logits;  // [B, Lv] sigmoid outputs of the forward pass
  const float* pred_spans;   // [B, Lv, 2] (-sigmoid, +sigmoid)
  const uint16_t* h_cls;     // [B*(Lv+1)+2, d] hidden activations (conv layout)
  const uint16_t* h_span;
  const float* w_cls;        // [3][d] packed fp32 weights (as in the forward)
  const float* w_span;       // [2][3][d]
  float* dz;                 // [B*(Lv+1)+2, 4] scratch: pre-sigmoid gradients (class, span0, span1, unused), conv layout
  uint16_t* dh_cls;          // [B*(Lv+1)+2, d] gradient w.r.t. the hidden activations (ReLU mask applied), bf16
  uint16_t* dh_span;
  float* gw_cls;             // parameter gradients in the reference layout: class_embed.layers.2.weight [1, d, 3]
  float* gb_cls;             // [1]
  float* gw_span;            // span_embed.layers.2.weight [2, d, 3]
  float* gb_span;            // [2]
  float* cs_cls;             // [d] column sums of dh_cls (bias gradient of conv layer 1) or null
  float* cs_span;
  float in_scale;            // loss scale applied to the incoming output gradients (all downstream gradients are scaled)
  float pgrad_scale;         // 1 / loss-scale for the parameter gradients written here
  int B, Lv, d, fmt_act, fmt_grad;
};
int launch_head_final_bwd(const HeadFinalBwdArgs& a, cudaStream_t stream);

// ---- weighted pool backward + assembly of the projector-output gradients ----
struct PoolBwdArgs {
  const float* x_txt;      // [B, Lt, d] projected text tokens
  const float* alpha;      // [B, Lt] softmax weights saved by the forward
  const float* w;          // [d]
  const float* g_pooled;   // [B, d] dL/d txt_mem_proj
  float* dx_txt;           // [B, Lt, d] gradient w.r.t. the projected text tokens (written, not accumulated)
  float* gw;               // [d] weightedpool.weight gradient (atomically accumulated, unscaled)
  float out_scale;         // loss scale applied to dx_txt
  int B, Lt, d;
};
int launch_pool_bwd(const PoolBwdArgs& a, cudaStream_t stream);

// out16[b*Ls + l, :] = cvt(dx_stream[b*L + off + l, :] + extra[b*Ls + l, :]); colsum += column sums (bias + type-embedding grads)
int launch_stream_gather(const float* dx_stream, int L, int off, const float* extra, float extra_scale, uint16_t* out16,
                         float* colsum, float colsum_scale, int B, int Ls, int d, int fmt, cudaStream_t stream);

// Backward of the learned text positions (rowops.h TxtPosArgs): one CTA per position l, looping over the samples.
//   g = drop(dpos[r]);  xhat = (xt[r] + table[l] - mean[r]) * rstd[r];  du = LayerNorm backward of g
//   dx[b*L + Lv + l] += du (stream gradient of x_t);  dtable[l] = pgrad_scale * sum_b du;  dgamma / dbeta += pgrad_scale * ...
struct TxtPosBwdArgs {
  const float* dpos;   // [B*Lt, d] gradient of pos_t (summed over the encoder layers; loss-scaled)
  const float* xt;     // [B*Lt, d] projected text tokens saved by the forward
  const float* table;  // [max_q_l, d]
  const float* gamma;  // [d]
  const float* mean;   // [B*Lt]
  const float* rstd;
  const float* mul32;  // [B*Lt, d] dropout multipliers of the forward, or null
  DropSpec drop;       // in-kernel regeneration (drop.on; ignored with mul32)
  float* dx;           // [B*L, d] stream gradient (text rows accumulated)
  float* dtable;       // [max_q_l, d]: rows < Lt written
  float* dgamma;       // [d] atomically accumulated
  float* dbeta;
  float pgrad_scale;
  int B, Lt, L, Lv, d;
};
int launch_txt_pos_bwd(const TxtPosBwdArgs& a, cudaStream_t stream);

}  // namespace uv
