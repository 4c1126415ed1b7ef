// Argument blocks of the criterion kernels (loss.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace uv {

struct LossArgs {
  // model outputs
  const float* pred_logits;  // [B, Lv]
  const float* pred_spans;   // [B, Lv, 2]
  const float* xv;           // [B, Lv, d] vid_mem_proj
  const float* xt;           // [B, d]     txt_mem_proj
  // targets (reference main/dataset.py:1078-1098)
  const float* timestamp;    // [B, Lv, 2]
  const float* tmask;        // [B, Lv] timestamp_mask
  const float* window;       // [B, Lv] timestamp_window
  const float* span_gt;      // [B, Lv, 2] span_labels_nn
  const float* sal;          // [B, Lv] saliency_scores
  const int64_t* pos_idx;    // [B] saliency_pos_labels[:, 0] or null
  float eos_coef, temperature;
  int B, Lv, d;
  // outputs
  float* losses;      // [5]: loss_b, loss_g, loss_f, loss_s_inter, loss_s_intra
  float* g_spans_b;   // [B, Lv, 2] d loss_b / d pred_spans
  float* g_spans_g;   // [B, Lv, 2] d loss_g / d pred_spans
  float* g_logits_f;  // [B, Lv]    d loss_f / d pred_logits
  float* cos_in;      // [B, Lv] cos(xv[b,l], xt[b])
  float* vnorm;       // [B, Lv] max(|xv[b,l]|, 1e-8)
  float* tnorm;       // [B]     max(|xt[b]|, 1e-8)
  float* sim;         // [B, B]  cos(xv[b,pos_b], xt[b'])
  float* g_cos_in;    // [B, Lv] d loss_s_intra / d cos_in
  float* g_sim;       // [B, B]  d loss_s_inter / d sim
};
int launch_loss_forward(const LossArgs& a, cudaStream_t stream);

struct LossBwdArgs {
  const float* w;  // [5] device: upstream gradient of each loss
  const float* g_spans_b;
  const float* g_spans_g;
  const float* g_logits_f;
  const float* cos_in;
  const float* vnorm;
  const float* tnorm;
  const float* sim;
  const float* g_cos_in;
  const float* g_sim;
  const float* xv;
  const float* xt;
  const int64_t* pos_idx;
  int B, Lv, d;
  float* d_logits;  // [B, Lv]
  float* d_spans;   // [B, Lv, 2]
  float* d_xv;      // [B, Lv, d]
  float* d_xt;      // [B, d]
};
int launch_loss_backward(const LossBwdArgs& a, cudaStream_t stream);

// QFVS criterion (reference model/univtg_qfvs.py): outputs [B, Lv] flattened row-major to N = B * Lv positions.
struct QfvsLossArgs {
  const float* pred_logits;  // [N]
  const float* xv;           // [B, Lv, d] vid_mem_proj
  const float* xt;           // [B, d]     txt_mem_proj
  const float* vmask;        // [N] src_vid_mask of the outputs
  const uint8_t* mask_gt;    // [N] bool: position i is kept iff mask_gt[i]
  const float* sal;          // row 0 of targets saliency_scores; entry k pairs with the k-th kept position (k < count <= N)
  int has_pos;               // "saliency_pos_labels" in targets
  float temperature;
  int B, Lv, d;
  // outputs: losses [5] as LossArgs; the rest is the LossArgs scratch (g_spans_* zeroed, g_logits_f, cos_in, vnorm, tnorm,
  // g_cos_in written) so that the MR/HL backward kernels apply unchanged
  float* losses;
  float* g_spans_b;
  float* g_spans_g;
  float* g_logits_f;
  float* cos_in;
  float* vnorm;
  float* tnorm;
  float* g_cos_in;
};
int launch_qfvs_loss_forward(const QfvsLossArgs& a, cudaStream_t stream);
// loss_bwd_small + loss_bwd_vid + loss_bwd_txt with pos_idx = null; unlike launch_loss_backward, the saliency term is never
// skipped (the QFVS saliency loss needs no positive index)
int launch_qfvs_loss_backward(const LossBwdArgs& a, cudaStream_t stream);

}  // namespace uv
