// Argument blocks + launchers of the bandwidth-bound row kernels (rowops.cu) and the attention kernel (attention.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "philox.cuh"

namespace uv {

struct LnArgs {
  const float* in;  // [rows, ld_in] fp32
  int ld_in;
  const uint16_t* in16;  // alternative 16-bit input [rows, ld_in] (packed feature shards: fp16 / bf16 per in_fmt); `in` is then unused
  int in_fmt;
  const uint16_t* add16;  // optional 16-bit [rows, ld_add16] branch added to `in` before normalising (x + DropPath(branch))
  int ld_add16;
  float* sum_out;         // optional fp32 [rows, d]: the pre-normalisation sum (saved for LayerNorm backward)
  int rows, d;
  const float* gamma;
  const float* beta;
  float eps;
  int fmt;
  // token structure of the residual stream: row = b*L + l; rows with l < Lv are video clips (L == 0: unstructured)
  int L, Lv;
  float* out32;        // [rows, d] fp32 (may alias `in`)
  uint16_t* out16;     // [rows, ld16] 16-bit operand (columns d..ld16 zero-filled by the generic kernel)
  uint16_t* out16p;    // [rows, ld16] 16-bit(x + pos) for video rows, 16-bit(x) for text rows
  int ld16;
  const float* pos;    // [B*Lv, d] fp32 sine table (row b*Lv + l)
  const float* pos_txt;  // [B*Lt, d] fp32 learned text positions (row b*Lt + l - Lv) added to out16p's text rows, or null
  uint16_t* outc;      // conv-head layout: row 1 + b*(Lv+1) + l of a [B*(Lv+1)+2, d] buffer (video rows only)
  const float* mul32;  // [rows, d] multiplier applied to the 16-bit outputs only (input-dropout mask incl. 1/(1-p)), or null
  DropSpec drop;       // in-kernel input dropout (drop.on; ignored when mul32 is given): same multiplier semantics
  float* mean_out;     // [rows] (training)
  float* rstd_out;     // [rows]
  int split;           // 1: fp16x3 (fmt 0, inference): add16 is read and out16 / out16p / outc are written as hi / lo pairs
  long long lo;        // split: elements from each of those buffers to its lo plane
};
// Instantiation launch_layernorm routed a call to (kernel_used): vec<NV> keeps d = 128 NV in registers, block<EPT> takes
// d <= 128 EPT one row per CTA, block2 the wide projector input, generic any d; _TXT adds pos_txt; + LN_SPLIT for fp16x3.
enum LnKernel {
  LN_VEC8 = 0, LN_VEC4, LN_VEC2, LN_VEC8_TXT, LN_VEC4_TXT, LN_VEC2_TXT, LN_BLOCK8, LN_BLOCK24, LN_BLOCK8_TXT, LN_BLOCK24_TXT,
  LN_BLOCK2_12, LN_GENERIC, LN_SPLIT = 12, LN_NUM_KERNELS = 24
};
int launch_layernorm(const LnArgs& a, cudaStream_t stream, int* kernel_used = nullptr);

// Learned text positions (txt_position_embed, reference model/position_encoding.py:19-41), one warp per text row r = b*Lt + l:
//   pos[r] = drop(LayerNorm(xt[r] + table[l])) (eps 1e-5), and the text row b*L + Lv + l of xpos16 becomes 16-bit(xt[r] + pos[r])
struct TxtPosArgs {
  const float* xt;      // [B*Lt, d] projected text tokens incl. the token-type row (x_t: the text rows of the stream)
  const float* table;   // [max_q_l, d] position_embeddings.weight
  const float* gamma;   // [d]
  const float* beta;    // [d]
  const float* mul32;   // [B*Lt, d] dropout multipliers, or null
  DropSpec drop;        // in-kernel dropout (drop.on; ignored when mul32 is given)
  float* pos;           // [B*Lt, d] out
  float* mean_out;      // [B*Lt] (training) or null
  float* rstd_out;
  uint16_t* xpos16;     // [B*L, d] q/k operand of encoder layer 0
  int B, Lt, L, Lv, d, fmt;
  int split;            // 1: fp16x3 - xpos16 gets its lo plane too, `lo` elements after the hi plane
  long long lo;
};
int launch_txt_pos(const TxtPosArgs& a, cudaStream_t stream);

// pos [B*Lv, d] sine table + key_mask [B, Lv+Lt] = cat(vid_mask, txt_mask)
// dp_out (optional): [dp_sites, B] DropPath scales floor(keep + u) / keep drawn in-kernel from (dp_seed, site * B + b)
int launch_sine_pos(const float* mask, const float* txt_mask, const float* dim_t, float* pos, float* key_mask, int B, int Lv,
                    int Lt, int d, cudaStream_t stream, float* dp_out = nullptr, int dp_sites = 0, unsigned long long dp_seed = 0,
                    float dp_keep = 1.f, const unsigned long long* dp_seed_ptr = nullptr);  // dp_seed_ptr: device seed (null: dp_seed)
// standalone generators (parity tests read the in-kernel draws back through them)
int launch_dropout_mask(const DropSpec& spec, size_t n, size_t cols, float* out, cudaStream_t stream);  // [n / cols, cols] row-major
int launch_droppath_scales(unsigned long long seed, int n, float keep, float* out, cudaStream_t stream,
                           const unsigned long long* seed_ptr = nullptr);
// *counter += 1; *seed = rng_seed_at(base, *counter)  (one thread; the head of a captured train step)
int launch_rng_advance(unsigned long long base, unsigned long long* counter, unsigned long long* seed, cudaStream_t stream);

struct PoolSalArgs {
  const float* x_txt;     // [B, Lt, d] projected text tokens (incl. token-type embedding)
  const float* x_vid;     // [B, Lv, d]
  const float* txt_mask;  // [B, Lt] 1 = valid
  const float* vid_mask;  // [B, Lv]
  const float* w;         // [d] weightedpool.weight
  float* pooled;          // [B, d]   (txt_mem_proj)
  float* saliency;        // [B, Lv]
  float* alpha_out;       // [B, Lt] softmax weights (training) or null
  float* logits_ws;       // [B, Lt] scratch
  int B, Lt, Lv, d;
};
int launch_pool_saliency(const PoolSalArgs& a, cudaStream_t stream);

struct HeadFinalArgs {
  const uint16_t* h_cls;   // [B*(Lv+1)+2, d] hidden of class_embed layer 2 (conv layout)
  const uint16_t* h_span;  // same for span_embed
  const float* w_cls;      // [3][d]     w_cls[t][c]  = class_embed.layers.2.weight[0, c, t]
  const float* w_span;     // [2][3][d]  w_span[o][t][c] = span_embed.layers.2.weight[o, c, t]
  const float* b_cls;      // [1]
  const float* b_span;     // [2]
  float* pred_logits;      // [B, Lv, 1]
  float* pred_spans;       // [B, Lv, 2]
  int B, Lv, d, fmt;
  int split;               // 1: fp16x3 - h_cls / h_span are hi / lo pairs, the lo planes `lo` elements after the hi planes
  long long lo;
};
int launch_conv_head_final(const HeadFinalArgs& a, cudaStream_t stream);

struct AttnArgs {
  // qkv: [B*L, 3d] 16-bit row-major; column blocks [0,d) = Q, [d,2d) = K, [2d,3d) = V (heads = dh-wide sub-blocks).
  CUtensorMap tm_qkv;  // box {64, 128}, 128B swizzle
  float scale;         // 1/sqrt(dh), applied to Q K^T inside the softmax exponent
  const float* key_mask;  // [B, L] 1 = valid key (src_key_padding_mask is its negation)
  uint16_t* out;          // [B*L, d] 16-bit attention output (heads concatenated)
  float* lse;             // [B, H, L] log-sum-exp per query row (training) or null
  int B, L, H, dh, d, fmt;
  DropSpec drop;          // attention dropout (drop.on; stream = encoder layer): P o M feeds P V, the row sum and lse stay un-dropped
  int split;              // 1: fp16x3 (fmt 0, no dropout): qkv and out are hi / lo pairs; tm_qkv is then a make_tmap_split pair
  long long lo_qkv, lo_out;  // split: elements from qkv / out to their lo planes
  int causal;             // 1: query i attends to keys j <= i only (dh = 64, tensor cores, no dropout, no split)
};
// Instantiation a launch ran (kernel_used): ATT_TC + 4 (dh == 128) + 2 bf16 + dropout, the causal kernel per format, the fp16x3
// kernel per head size, and the three SIMT kernels.
enum AttnKernel { ATT_TC = 0, ATT_CAUSAL = 8, ATT_SPLIT64 = 10, ATT_SPLIT128 = 11, ATT_SIMT = 12, ATT_SIMT_DROP = 13, ATT_SIMT_SPLIT = 14,
                  ATT_NUM_KERNELS = 15 };
int launch_attention(const AttnArgs& a, cudaStream_t stream, int* kernel_used = nullptr);
// SIMT variant for head sizes outside {64,128}; reads qkv through a plain pointer.
int launch_attention_simt(const AttnArgs& a, const uint16_t* qkv, cudaStream_t stream, int* kernel_used = nullptr);
// out [B, H, L, L] f32: the attention-dropout multipliers of `spec` (row = query, column = key), as the kernels apply them
int launch_attention_dropout_mask(const DropSpec& spec, int B, int H, int L, float* out, cudaStream_t stream);

}  // namespace uv
