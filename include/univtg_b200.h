/*
 * univtg_b200 — C ABI of the H100-native UniVTG hot path (cross-modal encoder + heads).
 *
 * Drop-in boundary: the reference reaches this path through ONE Python plugin call,
 *     importlib.import_module('model.' + opt.model_id).build_model(opt) -> (model, criterion)
 *     (reference main/config.py:341-342), then model(**model_inputs) (main/inference_mr.py:101,
 *     main/train_vlp_ddp.py:56) and criterion(outputs, targets) (main/train_vlp_ddp.py:57).
 * The reference has no FFI of its own (it is pure Python on torch); the functions below are what a
 * ctypes binding for that plugin binds (see INTEGRATION.md, univtg_b200/_lib.py).  Plain pointers and
 * sizes only: no torch types.  All pointers are DEVICE pointers unless stated otherwise, all tensors are
 * row-major/contiguous, `stream` is a cudaStream_t passed as void*.  Every function returns 0 on success,
 * non-zero on failure; univtg_last_error() then describes the failure (thread local).
 * Nothing here allocates device memory: the caller owns `packed` and `workspace`.
 */
#ifndef UNIVTG_B200_H_
#define UNIVTG_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UNIVTG_ABI_VERSION 2
#define UNIVTG_ADAMW_SCRATCH_FLOATS 2048

/* Model hyper-parameters: the fields of `args` that reference model/univtg.py:409-450 (build_model),
 * model/transformer_encoder_droppath.py:141-152 (build_transformer) and model/position_encoding.py:113-126 read. */
typedef struct univtg_config {
  int32_t hidden_dim;       /* args.hidden_dim  (d)            */
  int32_t nheads;           /* args.nheads      (H), dh = d/H  */
  int32_t dim_feedforward;  /* args.dim_feedforward            */
  int32_t enc_layers;       /* args.enc_layers                 */
  int32_t n_input_proj;     /* args.n_input_proj in {1,2,3}    */
  int32_t v_feat_dim;       /* args.v_feat_dim (already +2 TEF)*/
  int32_t t_feat_dim;       /* args.t_feat_dim                 */
  int32_t operand_format;   /* 0 = fp16 MMA operands (default), 1 = bf16; accumulation/LN/softmax/heads are fp32.
                             * 2 = fp16x3 (inference only): every 16-bit buffer holds hi = fp16(v) and a lo plane fp16(v - hi),
                             * and every product is A_hi B_hi + A_lo B_hi + A_hi B_lo.  The packed weights and the inference
                             * workspace are then twice their format-0 size: the first half is the format-0 layout (hi planes),
                             * and the lo plane of each 16-bit buffer lies exactly half the buffer size after its hi plane
                             * (the fp32 entries of the second half are unused).  univtg_prepare_workspace zeroes the separator
                             * rows of both planes.  univtg_forward_train, univtg_backward, univtg_train_workspace_bytes,
                             * univtg_adamw_step and the backward-only univtg_op_* entry points refuse it. */
} univtg_config;

/* Problem shape of one batch (reference Model.forward arguments, model/univtg.py:105). */
typedef struct univtg_shape {
  int32_t batch;  /* B   */
  int32_t l_vid;  /* L_v */
  int32_t l_txt;  /* L_t */
  int32_t training; /* 1: keep the activations backward needs (larger workspace) */
} univtg_shape;

/* Train-mode randomness generated inside the kernels (Philox4x32-10 keyed by (seed, mask index); csrc/philox.cuh): input
 * dropout of every LinearLayer (reference model/univtg.py:394,401) and DropPath (transformer_encoder_droppath.py:154-167).
 * The same struct passed to univtg_forward_train and univtg_backward reproduces the same draws; explicit multiplier tensors
 * (droppath_scale / drop_masks arguments) take precedence where given. */
typedef struct univtg_rng {
  uint64_t seed;        /* one value per training forward */
  float input_dropout;  /* args.input_dropout (p of nn.Dropout); 0 = off */
  float droppath;       /* args.droppath (drop probability); 0 = off */
} univtg_rng;

typedef struct univtg_plan univtg_plan; /* opaque; host memory only (shape, tile widths, buffer pointers) */

const char* univtg_last_error(void);
int univtg_abi_version(void);

/* Number of fp32 parameter tensors univtg_pack_weights expects, in this order (reference state_dict names):
 *   for i < n_input_proj: input_vid_proj.i.{LayerNorm.weight, LayerNorm.bias, net.1.weight, net.1.bias}
 *   for i < n_input_proj: input_txt_proj.i.{...same...}
 *   token_type_embeddings.weight
 *   for l < enc_layers: transformer.encoder.layers.l.{self_attn.in_proj_weight, self_attn.in_proj_bias,
 *        self_attn.out_proj.weight, self_attn.out_proj.bias, linear1.weight, linear1.bias, linear2.weight,
 *        linear2.bias, norm1.weight, norm1.bias, norm2.weight, norm2.bias}
 *   span_embed.layers.{0,1,2}.{weight,bias}; class_embed.layers.{0,1,2}.{weight,bias}; weightedpool.weight */
int univtg_num_params(const univtg_config* cfg);
/* Bytes of the packed-weight buffer (16-bit K-padded GEMM operands + fp32 vectors). */
size_t univtg_packed_bytes(const univtg_config* cfg);
/* Convert/re-layout the fp32 parameters into `packed` (device). `params`: HOST array of device pointers. */
int univtg_pack_weights(const univtg_config* cfg, const float* const* params, int32_t n_params, void* packed, void* stream);

/* Workspace bytes for one (config, shape). */
size_t univtg_workspace_bytes(const univtg_config* cfg, const univtg_shape* shape);
/* Zero the few regions of a workspace that kernels rely on reading as zeros (the separator rows of the conv-head buffers that
 * implement Conv1d's zero padding, reference model/univtg.py:375-377); everything else is written before it is read.  Call it
 * when a workspace buffer is used for the first time or handed over from another shape (workspaces may be pooled and shared
 * between shapes: size them for the largest shape).  training_ws: 0 = workspace of univtg_plan_create (univtg_workspace_bytes),
 * 1 = training workspace (univtg_train_workspace_bytes). */
int univtg_prepare_workspace(const univtg_config* cfg, const univtg_shape* shape, void* workspace, int32_t training_ws, void* stream);
/* Build a plan for one shape over `packed` and `workspace` (both must stay alive and must not move).
 * `dim_t`: device fp32 [hidden_dim], the sine-embedding denominators temperature**(2*(j//2)/d)
 * (reference model/position_encoding.py:75) evaluated by the caller.  Calls univtg_prepare_workspace on `stream`. */
int univtg_plan_create(const univtg_config* cfg, const univtg_shape* shape, const void* packed, void* workspace,
                       const float* dim_t, void* stream, univtg_plan** out);
void univtg_plan_destroy(univtg_plan* plan);

/* Element type of the src_txt / src_vid pointers the forward entry points (and univtg_backward) receive for this plan:
 * 0 = f32 (what the reference collate produces, default), 1 = fp16, 2 = bf16 (packed feature shards, univtg_b200/data.py: the CLIP /
 * SlowFast features are stored as 16-bit on disk, so the H2D copy and the first LayerNorm's read halve).  Masks stay f32. */
int univtg_plan_set_input_format(univtg_plan* plan, int32_t fmt);

/* Model.forward (reference model/univtg.py:105-155).
 *   src_txt [B,Lt,Dt] f32, src_txt_mask [B,Lt] f32 (1 = valid), src_vid [B,Lv,Dv] f32, src_vid_mask [B,Lv] f32
 *   droppath_scale: NULL (eval) or [2*enc_layers, B] f32 per-sample residual-branch scales
 *                   floor(keep + u)/keep in the reference's draw order (transformer_encoder_droppath.py:154-167)
 * outputs: pred_logits [B,Lv,1], pred_spans [B,Lv,2], vid_mem_proj [B,Lv,d], txt_mem_proj [B,1,d],
 *          saliency_scores [B,Lv]  (all f32) */
int univtg_forward(univtg_plan* plan, const float* src_txt, const float* src_txt_mask, const float* src_vid,
                   const float* src_vid_mask, const float* droppath_scale, float* pred_logits, float* pred_spans,
                   float* vid_mem_proj, float* txt_mem_proj, float* saliency_scores, void* stream);

/* ---- training (reference main/train_vlp_ddp.py:56-64: model(**inputs); criterion(outputs, targets); losses.backward()) ---- */

/* Bytes of the training workspace (saved activations + backward scratch) for one (config, shape). */
size_t univtg_train_workspace_bytes(const univtg_config* cfg, const univtg_shape* shape);
/* Model.forward in training mode: same outputs as univtg_forward, keeps what backward needs in `train_ws`.

 *   droppath_scale: NULL or [2*enc_layers, B] (see univtg_forward)
 *   drop_masks: NULL or HOST array of 2*n_input_proj device pointers (video layers, then text layers): fp32 [rows, din_i]
 *               input-dropout multipliers (0 or 1/(1-p)) drawn by the caller in the reference's order; entries may be NULL.
 *   rng: NULL or in-kernel randomness for whichever of the two is not given explicitly (mask index = position in drop_masks). */
int univtg_forward_train(univtg_plan* plan, void* train_ws, const float* src_txt, const float* src_txt_mask,
                         const float* src_vid, const float* src_vid_mask, const float* droppath_scale,
                         const float* const* drop_masks, const univtg_rng* rng, float* pred_logits, float* pred_spans,
                         float* vid_mem_proj, float* txt_mem_proj, float* saliency_scores, void* stream);
/* The multipliers univtg_forward_train draws for `rng`: mask `mask_index` ([rows, cols = din] row-major) and the DropPath
 * scales [n_sites = 2*enc_layers, batch].  Parity tests hand them to the oracle. */
int univtg_dropout_mask(const univtg_rng* rng, int32_t mask_index, size_t rows, size_t cols, float* out, void* stream);
int univtg_droppath_scales(const univtg_rng* rng, int32_t n_sites, int32_t batch, float* out, void* stream);
/* p of nn.MultiheadAttention's dropout (args.dropout) for the following univtg_forward_train / univtg_backward calls on this
 * plan; 0 = off (default).  The masks come from rng->seed (Philox, csrc/philox.cuh); p > 0 with rng == NULL is an error.
 * The value in effect at univtg_backward must be the one its forward ran with.  univtg_forward never applies it. */
int univtg_plan_set_attention_dropout(univtg_plan* plan, float p);
/* Seed source of the train-mode randomness of the following univtg_forward_train / univtg_backward calls on this plan (input
 * dropout, text-position dropout, attention dropout, DropPath): seed_dev = device uint64 read by every kernel that draws (once,
 * at its start) in place of rng->seed; NULL (default) = rng->seed.  The other rng fields (rates) still come from rng.  A CUDA
 * graph captured with a seed source draws new masks on every replay when univtg_rng_advance runs ahead of the step. */
int univtg_plan_set_seed_source(univtg_plan* plan, const uint64_t* seed_dev);
/* One-thread kernel: *counter_dev += 1; *seed_dev = univtg_rng_seed_at(base, *counter_dev) (splitmix64 sequence). */
int univtg_rng_advance(uint64_t base, uint64_t* counter_dev, uint64_t* seed_dev, void* stream);
/* HOST function: the k-th seed of the sequence of univtg_rng_advance (replay k of a graph with counter 0 before replay 1). */
uint64_t univtg_rng_seed_at(uint64_t base, uint64_t k);
/* The multipliers (0 or 1/(1-p)) the kernels apply in encoder layer `layer`: out [B, H, L, L] f32, row = query, column = key
 * (the reference's [B*H, L, L] layout).  Parity tests hand them to the oracle. */
int univtg_attention_dropout_mask(const univtg_rng* rng, float p, int32_t layer, int32_t B, int32_t H, int32_t L,
                                  float* out, void* stream);
/* Learned text positions (args.use_txt_pos; reference model/univtg.py:123, model/position_encoding.py:19-41): the text rows of
 * q = k = x + pos in every encoder layer get pos_t = Dropout(LayerNorm(x_t + P[l])) instead of zeros, where x_t is the projected
 * text token (token-type row included) and P the table.  The dropout is nn.Dropout(args.input_dropout) in training: in-kernel it
 * is input-dropout mask index 2*n_input_proj of rng (univtg_dropout_mask(rng, 2*n_input_proj, B*Lt, d) reads it back); an explicit
 * `drop_mul` takes precedence; univtg_forward never applies it.  univtg_plan_set_txt_pos(plan, NULL) switches the feature off
 * (the default); the setting in effect at univtg_backward must be the one its forward ran with, including the same scratch. */
typedef struct univtg_txt_pos {
  const float* table;     /* txt_position_embed.position_embeddings.weight [max_q_l, d]; read at every forward (not packed) */
  int32_t max_q_l;        /* rows of `table`: L_t > max_q_l is an error */
  const float* ln_weight; /* txt_position_embed.LayerNorm.weight [d] */
  const float* ln_bias;   /* txt_position_embed.LayerNorm.bias [d] */
  const float* drop_mul;  /* NULL or [B*L_t, d] dropout multipliers (0 or 1/(1-p)) of a training forward */
  void* scratch;          /* univtg_txt_pos_scratch_bytes(cfg, shape) bytes, owned by the caller; one per training forward
                           * whose backward is pending (it carries pos_t's statistics from the forward to the backward) */
} univtg_txt_pos;
int univtg_plan_set_txt_pos(univtg_plan* plan, const univtg_txt_pos* txt_pos);
/* Bytes of the scratch of univtg_txt_pos for (config, shape); shape->training selects the training layout. */
size_t univtg_txt_pos_scratch_bytes(const univtg_config* cfg, const univtg_shape* shape);

/* Backward of the last univtg_forward_train on (plan, train_ws).  g_*: upstream gradients of pred_logits [B,Lv,1],
 * pred_spans [B,Lv,2], vid_mem_proj [B,Lv,d], txt_mem_proj [B,1,d] (NULL = zero).  grads: HOST array of device pointers,
 * one ZERO-FILLED fp32 tensor per parameter in univtg_pack_weights order and in the parameter's own layout.
 * grad_scale: power-of-two loss scale S > 0.  Gradient GEMM operands share the plan's 16-bit format (one wgmma takes
 * A and B in one format); with fp16 operands the intermediate gradients are carried multiplied by S so they do not
 * underflow, and every parameter gradient is multiplied by 1/S where it is written (the results are unscaled).  Use 1 for
 * bf16 plans.  With text positions on (univtg_plan_set_txt_pos), n_grads is univtg_num_params + 3 and the last three tensors
 * are txt_position_embed.{position_embeddings.weight, LayerNorm.weight, LayerNorm.bias}; any other count is an error. */
int univtg_backward(univtg_plan* plan, void* train_ws, const float* src_txt, const float* src_vid, const float* droppath_scale,
                    const float* const* drop_masks, const univtg_rng* rng, const float* g_logits, const float* g_spans,
                    const float* g_vid_mem_proj, const float* g_txt_mem_proj, float grad_scale, float* const* grads,
                    int32_t n_grads, void* stream);

/* Gradient-exchange overlap (the reference relies on DistributedDataParallel's bucketed all-reduce overlapping backward,
 * main/train_vlp_ddp.py:272-275).  univtg_backward finalises parameter gradients in n = enc_layers + 3 stages:
 *   stage 0: conv heads + pooling weight; stage 1 + k: encoder layer enc_layers-1-k; stage n-2: projector weights / biases, the later
 *   projector layers' LayerNorm terms, token-type embedding; stage n-1: LayerNorm terms of the first projector layers (a few KB: the
 *   large input-projection gradients start their exchange before the backward's last kernels run).
 * univtg_backward_stages writes, per stage, two half-open parameter-index ranges {first0, last0, first1, last1}
 * (univtg_pack_weights order; an empty second range is 0,0) and returns n (ranges == NULL: just returns n).
 * univtg_plan_set_grad_events installs n cudaEvent_t handles; univtg_backward records event k on its stream as soon as stage
 * k's gradients are final, so a communication stream can wait on it and reduce that slice while the backward continues.
 * n = 0 removes them.  (enc_layers <= 16, so n <= 19.)  With text positions on, the three appended gradients (indices
 * univtg_num_params .. +3, not listed by univtg_backward_stages) are final at stage n-2. */
int univtg_backward_stages(const univtg_config* cfg, int32_t* ranges, int32_t max_stages);
/* The GEMM launches of univtg_backward are persistent grids of one CTA per SM.  When a collective (NCCL) runs beside the backward
 * its CTAs occupy some SMs; give the backward the number of SMs that are left (0 = all) so that its grids stay single-wave. */
int univtg_plan_set_backward_sm_budget(univtg_plan* plan, int32_t num_sms);
int univtg_plan_set_grad_events(univtg_plan* plan, void* const* events, int32_t n);

/* SetCriterion for model_id=univtg (reference model/univtg.py:195-282): losses5 = {loss_b, loss_g, loss_f, loss_s_inter,
 * loss_s_intra}.  targets as main/dataset.py:1078-1098 builds them (all f32 except saliency_pos_idx = saliency_pos_labels[:,0],
 * int64, NULL when absent).  `scratch` (univtg_loss_scratch_bytes) carries per-loss gradients to univtg_loss_backward. */
size_t univtg_loss_scratch_bytes(int32_t B, int32_t Lv);
int univtg_loss_forward(const float* pred_logits, const float* pred_spans, const float* vid_mem_proj, const float* txt_mem_proj,
                        const float* timestamp, const float* timestamp_mask, const float* timestamp_window,
                        const float* span_labels_nn, const float* saliency_scores, const int64_t* saliency_pos_idx, int32_t B,
                        int32_t Lv, int32_t d, float eos_coef, float temperature, float* losses5, void* scratch, void* stream);
/* w5: device fp32 [5] = dL/d(loss_k).  Writes the gradients of the four model outputs. */
int univtg_loss_backward(const float* w5, const float* vid_mem_proj, const float* txt_mem_proj, const int64_t* saliency_pos_idx,
                         int32_t B, int32_t Lv, int32_t d, const void* scratch, float* d_logits, float* d_spans,
                         float* d_vid_mem_proj, float* d_txt_mem_proj, void* stream);

/* SetCriterion for model_id=univtg_qfvs (reference model/univtg_qfvs.py:215-261, 358-377), query-focused video summarisation.
 * The outputs of one forward over B = max_segment_num segments of Lv = max_frame_num frames are read as N = B * Lv flat positions.
 * Position i is kept iff mask_gt[i] (bool bytes, [N]); the k-th kept position pairs with saliency_scores[k] (row 0 of the
 * targets, at least N entries; entries at or beyond the kept count are ignored).  losses5 as univtg_loss_forward:
 *   loss_f       = sum over kept of BCE(pred_logits, t) (logs clamped at -100) / sum(t)
 *   loss_s_intra = -mean over kept t > 0 of log softmax(z), over all kept positions; z = (cos(vid_mem_proj, txt_mem_proj)
 *                  + log(src_vid_mask + 1e-45)) / temperature, i.e. the model's saliency_scores / temperature
 *   loss_b = loss_g = loss_s_inter = 0.  loss_f and loss_s_intra are 0 when sum(t) == 0, loss_s_intra also when
 *   has_pos_labels == 0; their gradients are then 0.  No host synchronisation.  `scratch`: univtg_loss_scratch_bytes(B, Lv). */
int univtg_qfvs_loss_forward(const float* pred_logits, const float* vid_mem_proj, const float* txt_mem_proj, const float* src_vid_mask,
                             const uint8_t* mask_gt, const float* saliency_scores, int32_t has_pos_labels, int32_t B, int32_t Lv,
                             int32_t d, float temperature, float* losses5, void* scratch, void* stream);
/* w5: device fp32 [5] = dL/d(loss_k).  Writes d pred_logits [N], d vid_mem_proj [B, Lv, d] and d txt_mem_proj [B, d];
 * pred_spans gets no gradient.  Overwrites the span-gradient part of `scratch`. */
int univtg_qfvs_loss_backward(const float* w5, const float* vid_mem_proj, const float* txt_mem_proj, int32_t B, int32_t Lv,
                              int32_t d, void* scratch, float* d_logits, float* d_vid_mem_proj, float* d_txt_mem_proj, void* stream);

/* Number of kernels one univtg_forward launches (for bench accounting). */
int univtg_forward_num_launches(const univtg_plan* plan);
/* Kernels this library has launched since it was loaded (every launch of every entry point; memsets / memcpys not counted). */
int64_t univtg_launch_count(void);

/* Optional per-launch CUDA-event timeline of univtg_forward (bench / profiling only; adds event records to the stream).
 * read_profile returns the number of launches of the last forward and fills ms[i] / kinds[i]
 * (kind 0 = bandwidth-bound row kernel, 1 = tensor-core GEMM, 2 = attention); it synchronises on the last event. */
int univtg_plan_set_profiling(univtg_plan* plan, int32_t enable);
int univtg_plan_read_profile(univtg_plan* plan, float* ms, int32_t* kinds, int32_t cap);

/* ---- single operators (unit tests / profiling; same kernels the plan uses) ---- */

/* C[M,N] = act(A*B^T + bias) * alpha.  a: [M,K] (a_mn=0) or [K,M] (a_mn=1); b: [N,K] (b_mn=0) or [K,N] (b_mn=1),
 * 16-bit operands in `fmt`; K and the leading dimensions must be multiples of 8 elements.  out32 [M,N] f32 and/or
 * out16 [M,N] 16-bit.  bn: tile width, multiple of 16 in [32,256] (multiple of 64 when b_mn); ksplit>1 accumulates
 * atomically into a pre-zeroed out32. */
int univtg_op_gemm(const void* a, const void* b, int32_t M, int32_t N, int32_t K, int32_t a_mn, int32_t b_mn, int32_t fmt,
                   int32_t bn, int32_t ksplit, const float* bias, int32_t act, float alpha, float* out32, void* out16,
                   void* stream);
/* fmt = 2 (fp16x3) for univtg_op_gemm, univtg_op_layernorm and univtg_op_attention: every 16-bit argument is a hi plane
 * followed directly by its lo plane of the same shape (a: lo at a + M*K, b: b + N*K, out16: out16 + M*N; layernorm out16:
 * out16 + rows*ld16; attention qkv: qkv + B*L*3d, out: out + B*L*d).  The GEMM needs a_mn = b_mn = 0, N % 16 == 0,
 * 32-byte aligned outputs and lo planes, and no ksplit with out16. */
/* Same GEMM launched as 2-CTA clusters: vertically adjacent tiles share a K-major B tile through TMA multicast (half the
 * L2 -> SM traffic of B).  bn multiple of 32; b_mn must be 0 (an MN-major B is rejected with an error). */
int univtg_op_gemm_cluster(const void* a, const void* b, int32_t M, int32_t N, int32_t K, int32_t a_mn, int32_t b_mn,
                           int32_t fmt, int32_t bn, int32_t ksplit, const float* bias, int32_t act, float alpha, float* out32,
                           void* out16, void* stream);
/* One problem of univtg_op_gemm_group: C[M,N] = epilogue(sum_k A(m,k) B(n,k)) with the epilogue univtg_backward and the
 * training forward use.  16-bit formats: 0 fp16, 1 bf16, -1 = the group's `fmt`; A and B must resolve to the same format.
 *   conv = 0: a [M,K] (a_mn=0) or [K,M] (a_mn=1), b [N,K] (b_mn=0) or [K,N] (b_mn=1), pitches lda / ldb (multiples of 8).
 *   conv = 1: k=3 Conv1d data gradient in the conv-head layout (buffer row = logical row + 1, rows 0 and M+1 zero): a = dY
 *             [M+2, K] (K = out channels, multiple of 64), b = packed weight [K, 3N] with b[o, t*N + c] = W[o, c, t] (ldb = 3N);
 *             row m of the result is sum_t dY[m - t + 1] W[:, :, t].  a_mn = 0, b_mn = 1.
 *   conv = 2: weight gradient of tap `tap`: a = dY [K+2, M], b = X [K+2, N] (same layout); C[n, c] = sum_m dY[m, n] X[m + tap - 1, c]
 *             over the K logical rows.  a_mn = b_mn = 1.
 *   conv = 3: k=3 Conv1d forward of the heads over the same layout: a = X [M+2, K/3] (pitch lda; rows 0, M+1 and the separator rows
 *             zero), b = packed weight [N, K] with b[o, t*K/3 + c] = W[o, c, t] (ldb = K); row m of the result is
 *             sum_t X[m + t - 1] W[:, :, t] (logical rows).  a_mn = b_mn = 0, K/3 % 64 == 0, cluster 1.
 * Epilogue: v = act(acc + bias[n]) * alpha * row_scale[m / rps_in]; out row = (m / rps_in) * rps_out + m % rps_in + row_off
 * (identity when rps_in = 0); zero_sep stores v = 0 and skip_sep stores nothing on rows with m % rps_in == rps_in - 1;
 * v += resid[out row]; mask16 (indexed like out16, group fmt) zeroes v where mask16 <= 0, or multiplies v by it (mask_mul = 1);
 * out32 at out rows (accumulate = 1: out32 += v), out32_id at row m, out16 at out rows, out16p = 16-bit(v + addtab[m]) at out rows
 * (pitch ld16), dact16 = GELU'(acc + bias) with act = 2; colsum[n] += colsum_scale * sum of the stored v.  ksplit > 1 splits the K
 * loop into partial sums added into a pre-zeroed out32; ksplit > 1 and accumulate are rejected with act, resid, out16, out16p,
 * out32_id or dact16.  vec_ok is an output: 0 scalar, 1 128-bit, 2 256-bit epilogue accesses. */
typedef struct univtg_gemm_problem {
  const void* a;
  int32_t lda, a_mn;
  const void* b;
  int32_t ldb, b_mn;
  int32_t M, N, K, ksplit;
  int32_t a_fmt, b_fmt, out_fmt;
  int32_t conv, tap;
  const float* bias;
  int32_t act; /* 0 none, 1 ReLU, 2 GELU (erf) */
  float alpha;
  const float* row_scale;
  int32_t rps_in, rps_out, row_off, zero_sep, skip_sep;
  const float* resid;
  int32_t ld_resid;
  const float* addtab;
  int32_t ld_addtab;
  float* out32;
  int32_t ld32;
  float* out32_id;
  int32_t ld32_id;
  void* out16;
  void* out16p;
  int32_t ld16, accumulate;
  const void* mask16;
  int32_t ld_mask, mask_mul;
  void* dact16;
  int32_t ld_dact;
  float* colsum;
  float colsum_scale;
  int32_t vec_ok; /* written */
} univtg_gemm_problem;
/* 1 <= num <= 4 problems in one persistent launch (tiles interleaved over the SMs).  bn: tile width (multiple of 16 in [32,256];
 * of 64 when a B operand is MN-major); cluster = 2 launches 2-CTA clusters (K-major B only).  full (optional) receives 1 when the
 * FULL epilogue variant ran, 0 for the lean one. */
int univtg_op_gemm_group(univtg_gemm_problem* problems, int32_t num, int32_t fmt, int32_t bn, int32_t cluster, int32_t* full,
                         void* stream);

/* LayerNorm backward over rows (the kernels of univtg_backward):  xhat = (y - mean) * rstd, g = dout' * gamma with
 * dout' = dout * (dout_mul or the in-kernel dropout of (rng, mask_index), as univtg_dropout_mask reads it back),
 *   dy = rstd * (g - mean_j g - xhat * mean_j(g xhat)), zeroed where y <= 0 when relu_mask_y;  dy32 = dy;
 *   dbr16 = 16-bit(dy * row_scale[row / L]) with columns [d, ld16) set to 0;  dgamma += pgrad_scale * sum_rows dout' xhat;
 *   dbeta += pgrad_scale * sum_rows dout';  colsum += pgrad_scale * sum_rows dy * row_scale (fp32, before rounding).
 * With dy32 = dbr16 = NULL only the parameter gradients are formed, and y may be given as 16-bit (y16, y_fmt). */
typedef struct univtg_ln_bwd {
  const float* dout;
  int32_t ld_dout;
  const float* y;
  int32_t ld_y;
  const void* y16;
  int32_t y_fmt;
  const float* mean;
  const float* rstd;
  const float* gamma;
  int32_t rows, d;
  const float* row_scale;
  int32_t L, relu_mask_y;
  float* dy32;
  void* dbr16;
  int32_t ld16, fmt16;
  float* dgamma;
  float* dbeta;
  float* colsum;
  float pgrad_scale;
  const float* dout_mul;
} univtg_ln_bwd;
/* rng == NULL or rng->input_dropout == 0: no in-kernel dropout.  kernel_used (optional) receives the instantiation that ran:
 * 0 parameters only, 1/2/3 warp-per-row d = 256/512/1024, 4/5 128-bit d <= 512 / <= 1024, 6/7 row-per-block d <= 1024 / <= 3072. */
int univtg_op_layernorm_bwd(const univtg_ln_bwd* args, const univtg_rng* rng, int32_t mask_index, int32_t* kernel_used, void* stream);

/* Last conv layer of the heads, backward (d % 8 == 0; activations in the conv-head layout [B*(Lv+1)+2, d], fmt_act):
 *   dz = pre-sigmoid gradients * in_scale [B*(Lv+1)+2, 4] (scratch, written); dh_cls / dh_span = ReLU'(h) * conv-transpose of dz
 *   (fmt_grad, separator rows 0); gw_* ([o, d, 3]), gb_*, cs_* (column sums of dh_*, both or neither) += pgrad_scale * ... */
typedef struct univtg_head_final_bwd {
  const float* g_logits;
  const float* g_spans;
  const float* pred_logits;
  const float* pred_spans;
  const void* h_cls;
  const void* h_span;
  const float* w_cls;  /* [3][d] */
  const float* w_span; /* [2][3][d] */
  float* dz;
  void* dh_cls;
  void* dh_span;
  float* gw_cls;
  float* gb_cls;
  float* gw_span;
  float* gb_span;
  float* cs_cls;
  float* cs_span;
  float in_scale, pgrad_scale;
  int32_t B, Lv, d, fmt_act, fmt_grad;
} univtg_head_final_bwd;
int univtg_op_head_final_bwd(const univtg_head_final_bwd* args, void* stream);
/* colsum[c] += scale * sum_r in16[r, c] (the stored 16-bit values).  txt16 != NULL also copies the text rows (r % L >= Lv) of the
 * first txt_cols columns into txt16 [rows / L * (L - Lv), txt_cols].  cols, ld, txt_cols multiples of 8, pointers 16-byte aligned. */
int univtg_op_colsum16(const void* in16, int32_t ld, int32_t rows, int32_t cols, int32_t fmt, float* colsum, float scale, void* txt16,
                       int32_t L, int32_t Lv, int32_t txt_cols, void* stream);
/* out16 = 16-bit(in32); colsum (optional) += colsum_scale * column sums of in32 (fp32, before rounding); txt16 as above.
 * cols, pitches, txt_cols multiples of 4; in32 16-byte, out16 / txt16 8-byte aligned. */
int univtg_op_cvt16_colsum(const float* in32, int32_t ld_in, void* out16, int32_t ld_out, int32_t rows, int32_t cols, int32_t fmt,
                           float* colsum, float colsum_scale, void* txt16, int32_t L, int32_t Lv, int32_t txt_cols, void* stream);
/* out16[b*Ls + l] = 16-bit(dx[b*L + off + l] + extra_scale * extra[b*Ls + l]) (extra optional), colsum (optional) += colsum_scale *
 * column sums of the fp32 values.  d % 4 == 0, off + Ls <= L, dx / extra 16-byte and out16 8-byte aligned. */
int univtg_op_stream_gather(const float* dx, int32_t L, int32_t off, const float* extra, float extra_scale, void* out16, float* colsum,
                            float colsum_scale, int32_t B, int32_t Ls, int32_t d, int32_t fmt, void* stream);
/* Weighted-pool backward: pooled = sum_l alpha_l x_l; dx_txt [B,Lt,d] = out_scale * (alpha g + dlogit w) (written);
 * gw [d] += sum dlogit x (unscaled). */
int univtg_op_pool_bwd(const float* x_txt, const float* alpha, const float* w, const float* g_pooled, float* dx_txt, float* gw,
                       float out_scale, int32_t B, int32_t Lt, int32_t d, void* stream);
/* Learned text positions backward (d <= 1024): g = dpos * (mul32 or the dropout of (rng, mask_index)); LayerNorm backward of
 * u = xt + table[l] with the given mean / rstd; dx[b*L + Lv + l] += du; dtable rows < Lt = pgrad_scale * sum_b du (written);
 * dgamma / dbeta += pgrad_scale * ... */
typedef struct univtg_txt_pos_bwd {
  const float* dpos;
  const float* xt;
  const float* table;
  const float* gamma;
  const float* mean;
  const float* rstd;
  const float* mul32;
  float* dx;
  float* dtable;
  float* dgamma;
  float* dbeta;
  float pgrad_scale;
  int32_t B, Lt, L, Lv, d;
} univtg_txt_pos_bwd;
int univtg_op_txt_pos_bwd(const univtg_txt_pos_bwd* args, const univtg_rng* rng, int32_t mask_index, void* stream);
/* Profiling aid: when `buf` (device, >= num_SMs*8 uint64) is non-NULL every following GEMM launch stamps %globaltimer per CTA:
 * [0] entry, [1] setup done, [2] all TMA issued, [3] first stage landed, [4] last MMA of the first tile retired, [5] unused,
 * [6] epilogue done, [7] exit.  Pass NULL to switch it off. */
int univtg_debug_gemm_timeline(void* buf);
/* Host-only: the tile width / split-K factor the GEMM launcher's cost model picks for a grouped launch (num <= 4 problems of
 * M x N with kblocks 64-wide k-blocks each; step 16 for K-major B, 64 for MN-major B).  Testing / tuning aid. */
int univtg_debug_choose_tile(const int32_t* Ms, const int32_t* Ns, const int32_t* kblocks, int32_t num, int32_t num_sms, int32_t step,
                             int32_t max_split, int32_t* bn, int32_t* ksplit);
/* Host-only, the same with a split limit per problem (powers of two; 1 for a problem whose epilogue cannot accumulate): the
 * launch's one tile width and each problem's split-K factor (ksplit[num]).  univtg_debug_choose_tile gives every problem the
 * limit max_split and reports the largest factor. */
int univtg_debug_choose_tile_group(const int32_t* Ms, const int32_t* Ns, const int32_t* kblocks, const int32_t* max_split, int32_t num,
                                   int32_t num_sms, int32_t step, int32_t* bn, int32_t* ksplit);
/* Host-only: the static deal of a grouped GEMM launch's work units (output tile x k-split) over its persistent CTAs, walked as
 * the kernel's CTAs walk it.  Units are numbered problem by problem (tiles n fastest, then m, then the split); cta[u] receives
 * the CTA that runs unit u, -1 if none does and -2 if more than one does.  Returns the number of units (cap bounds what is
 * written), or -1 for bad arguments. */
int32_t univtg_debug_gemm_deal(const int32_t* Ms, const int32_t* Ns, const int32_t* kblocks, const int32_t* ksplit, int32_t num,
                               int32_t num_sms, int32_t bn, int32_t* cta, int32_t cap);
/* Parameter update of the reference's training loop (main/train_vlp_ddp.py:66-68 = main/train_mr.py:64-66; optimizer built at
 * main/config.py:350 as torch.optim.AdamW(lr, weight_decay)) over ONE flat fp32 buffer of n floats (n % 4 == 0, 16-byte
 * aligned; the plugin lays every parameter and its gradient out at the same offsets):
 *   total_norm = ||grads||_2;  if max_grad_norm > 0: g *= min(1, max_grad_norm / (total_norm + 1e-6))   (clip_grad_norm_)
 *   p *= 1 - lr*wd;  m = m + (1-beta1)(g - m);  v = beta2 v + (1-beta2) g^2;
 *   p -= lr/(1-beta1^step) * m / (sqrt(v)/sqrt(1-beta2^step) + eps)                                      (AdamW, step >= 1)
 * scratch3: device fp32 [UNIVTG_ADAMW_SCRATCH_FLOATS] (per-block partial sums of squares live behind the first four floats: the
 * norm is accumulated in a fixed order, without atomics, so the update is bit-reproducible and identical on every data-parallel
 * rank); on return [1] holds total_norm (what clip_grad_norm_ returns) and [2] is 1.0 when total_norm was not
 * finite - then NOTHING was updated (the skipped step of dynamic loss scaling; the fp16 gradient operands of univtg_backward can
 * overflow when grad_scale is too large), else 0.0.  write_clipped_grads != 0 also stores the clipped gradients back
 * (clip_grad_norm_ scales .grad in place).
 * cfg + packed (both non-NULL; the flat buffers must then start with the config's parameters in univtg_pack_weights order, each
 * padded to a multiple of 4 floats; floats beyond them - the text-position tensors of univtg_backward - are parameters without a
 * 16-bit copy and are updated like the rest): the kernel also refreshes the 16-bit copies of the GEMM weight matrices inside `packed` from the
 * values it has just computed, so no separate re-packing pass re-reads the weights; call univtg_pack_vectors afterwards for the
 * fp32 vectors (LayerNorm terms, biases, token-type rows - a few hundred KB). */
int univtg_adamw_step(float* params, float* grads, float* exp_avg, float* exp_avg_sq, size_t n, float lr, float beta1,
                      float beta2, float eps, float weight_decay, int32_t step, float max_grad_norm,
                      int32_t write_clipped_grads, float* scratch3, const univtg_config* cfg, void* packed, void* stream);
/* univtg_adamw_step with the optimizer state in device memory, for CUDA-graph replay: lr_dev = device fp32 learning rate;
 * step_dev = device int32 count of completed updates - this update runs at step *step_dev + 1 and writes that value back only
 * when it was not skipped (scratch3[2] == 0); bc_table = device fp32 [table_len][2] holding (bc1, bc2_sqrt) of steps 1 ..
 * table_len as univtg_adamw_bias_table writes them (steps past table_len reuse the last row: build it with
 * univtg_adamw_bias_table_len rows, after which both terms are 1.0f for good).  With that table the update is bit-identical to
 * univtg_adamw_step at the same step.  scratch3[3] is used as well (the staged step). */
int univtg_adamw_step_dev(float* params, float* grads, float* exp_avg, float* exp_avg_sq, size_t n, const float* lr_dev,
                          float beta1, float beta2, float eps, float weight_decay, int32_t* step_dev, float max_grad_norm,
                          int32_t write_clipped_grads, float* scratch3, const univtg_config* cfg, void* packed,
                          const float* bc_table, int32_t table_len, void* stream);
/* HOST functions: rows t = 1 .. len of the bias-correction table, out_host [len][2] = ((float)(1 - beta1^t),
 * (float)sqrt(1 - beta2^t)) in double precision (univtg_adamw_step's expressions); and the number of rows after which both
 * terms stay 1.0f (0 with an error message for betas outside [0, 1) or a table longer than 2^26 rows). */
int univtg_adamw_bias_table(float beta1, float beta2, int32_t len, float* out_host);
int32_t univtg_adamw_bias_table_len(float beta1, float beta2);
/* univtg_pack_weights restricted to the fp32 vectors and the two tiny last-conv tensors (everything that is not a 16-bit matrix). */
int univtg_pack_vectors(const univtg_config* cfg, const float* const* params, int32_t n_params, void* packed, void* stream);

/* HOST function (no device work): assemble one padded batch from a memory-mapped 16-bit feature shard into (pinned) staging
 * buffers - what the reference's per-sample loads + pad_sequences_1d collate do (main/dataset.py:644-696, 1037-1052,
 * utils/tensor_utils.py:6-53).  src_vid [rows, Dv] / src_txt [rows, Dt]: the shard's 16-bit matrices; sample b copies vid_len[b]
 * rows starting at vid_row0[b] (txt likewise) into dst_vid [B, Lv, Dv] / dst_txt [B, Lt, Dt], zero-fills the rest and writes the
 * float masks dst_vmask [B, Lv] / dst_tmask [B, Lt] (1 = valid).  threads > 1 uses a persistent worker pool. */
int univtg_host_assemble_batch(void* dst_vid, void* dst_txt, float* dst_vmask, float* dst_tmask, const void* src_vid,
                               const void* src_txt, const int64_t* vid_row0, const int64_t* txt_row0, const int32_t* vid_len,
                               const int32_t* txt_len, int32_t B, int32_t Lv, int32_t Lt, int32_t Dv, int32_t Dt, int32_t threads);

/* Direct variant: page-lock the shard's memory mapping once (univtg_host_register; enable = 0 undoes it) and let the copy engines
 * pull every sample's rows straight from it into the device batch on `stream` - no CPU staging copy.  mask_stage: pinned host
 * scratch of B * (Lv + Lt) floats that must stay untouched until the stream has passed this call. */
int univtg_host_register(void* base, size_t bytes, int32_t enable);
int univtg_h2d_gather_batch(void* dev_vid, void* dev_txt, float* dev_vmask, float* dev_tmask, float* mask_stage, const void* src_vid,
                            const void* src_txt, const int64_t* vid_row0, const int64_t* txt_row0, const int32_t* vid_len,
                            const int32_t* txt_len, int32_t B, int32_t Lv, int32_t Lt, int32_t Dv, int32_t Dt, void* stream);

/* Post-forward decode of the reference's MR evaluation loop, on the device (SURVEY.md section 8 rows a16 / f-1).
 * univtg_decode_mr = main/inference_mr.py:112-120,146-157 (and main_gradio.py:100-106 with duration == NULL):
 *   score = pred_logits[b,l] (0 where timestamp_mask[b,l] == 0); (st, ed) = (timestamp + pred_spans)[b,l] * duration[b], clamped to
 *   [0, duration[b]] (no scaling / clamping when duration == NULL); rows [st, ed, score] sorted by score, descending, ties in clip
 *   order (Python's stable sort) when sort != 0.  windows [B,Lv,3] f32 receives the rows, windows_r4 [B,Lv,3] f64 (optional) the
 *   same numbers rounded like float(f"{e:.4f}") (exact), order [B,Lv] (optional) the source clip index of every row.  Lv <= 4096.
 * univtg_temporal_nms = utils/temporal_nms.py:25-74 as called by main/inference_mr.py:31-40: per sample, the first
 *   min(n, max_before_nms) rows of windows [B,n,3] f64 (sorted by score) go through greedy NMS with the reference's
 *   intersection / convex-hull "IoU" > nms_thd test in IEEE double; out [B,max_after_nms,3] f64, counts [B] rows kept. */
int univtg_decode_mr(const float* pred_logits, const float* pred_spans, const float* timestamp, const float* timestamp_mask,
                     const float* duration, int32_t B, int32_t Lv, int32_t sort, float* windows, double* windows_r4, int32_t* order,
                     void* stream);
int univtg_temporal_nms(const double* windows, int32_t B, int32_t n, int32_t max_before_nms, double nms_thd, int32_t max_after_nms,
                        double* out, int32_t* counts, void* stream);

/* The evaluation epoch's variants (main/inference_mr.py:101-222): one ragged row pool per epoch, query q owning the Lv rows of its
 * batch (each batch is padded to its own maximum) from pool row offsets[q].
 * univtg_decode_mr_pool = univtg_decode_mr writing the rounded rows of sample b to rows [*,3] f64 at row row_offset + b * Lv, and:
 *   hl (with saliency_scores [B,Lv]): the highlight value of every clip at hl[row_offset + b * Lv + l], fp32(fp16(saliency)), or with
 *     add_prob != 0 (eval_mode "add", :124-125) fp32(fp16(saliency)) + prob, prob being pred_logits with 0 where timestamp_mask == 0;
 *   valid_len (with src_vid_mask [B,Lv]): src_vid_mask.sum(1) as int at valid_len[sample_offset + b];
 *   round_multiple > 0 (eval/postprocessing.py:26-51): st / ed become double(rintf(fp32(x) / clip_length) * clip_length) in fp32
 *     (IEEE division, ties to even) and the score float(f"{fp32(score):.4f}").  clip_length > 0.
 * univtg_temporal_nms_pool = univtg_temporal_nms over that pool: query q's rows are row_offsets[q] .. row_offsets[q + 1] - 1
 *   (row_offsets [Q+1] i64 on the device, at most max_rows each); with sort != 0 the first max_before_nms rows are first sorted by
 *   score (descending, ties in row order) as temporal_nms does for clip-order (--no_sort_results) rows. */
int univtg_decode_mr_pool(const float* pred_logits, const float* pred_spans, const float* timestamp, const float* timestamp_mask,
                          const float* duration, const float* saliency_scores, const float* src_vid_mask, int32_t B, int32_t Lv,
                          int32_t sort, int32_t add_prob, int32_t round_multiple, float clip_length, int64_t row_offset,
                          int64_t sample_offset, double* rows, float* hl, int32_t* valid_len, void* stream);
int univtg_temporal_nms_pool(const double* rows, const int64_t* row_offsets, int32_t Q, int32_t max_rows, int32_t max_before_nms,
                             double nms_thd, int32_t max_after_nms, int32_t sort, double* out, int32_t* counts, void* stream);

/* Per-query metrics of the reference's eval_submission (eval/eval.py:20-289, eval/utils.py:17-211), IEEE double, equal to numpy's
 * values bit for bit; univtg_b200/metrics.py does the packing and the means over queries.
 * univtg_eval_mr: pred [Q,10,3] f64 = the first n_pred[q] (1..10) rows [st, ed, score] of each query in submission order;
 *   gt [Q,G,2] f64 = the n_gt[q] (1..G) gt windows, G <= 64.  For the ranges r = 0 (0,10], 1 (10,30], 2 (30,inf), 3 full
 *   (get_data_by_range's length filter): kept [4,Q] = 1 when the query has a gt window in the range; then ap [4,Q,10] =
 *   compute_average_precision_detection at IoU 0.50:0.05:0.95 (gt windows visited NaN first, then decreasing IoU, ties to the
 *   higher index), iou_r1 [4,Q] and iou_r5 [4,Q] = the paired IoUs of compute_mr_r1 / compute_mr_r5.  Rows not kept are 0.
 * univtg_eval_hl: sal [Q,S] f64 = the n_sal[q] (>= 1) predicted saliency scores, zero padded; labels [Q,C] bit (3*l + a) =
 *   (score of annotator a >= 2 + l) over the n_clips[q] = int(duration / 2) clips (1..C, C <= 4096); scratch [Q,9,C] f64.
 *   ap [3,Q,3] = get_ap(labels, sal cut / zero-padded to n_clips) (scikit-learn precision_recall_curve); hit [3,Q,3] = the label
 *   at np.argmax of the whole predicted list (0 when that index is >= n_clips). */
int univtg_eval_mr(const double* pred, const int32_t* n_pred, const double* gt, const int32_t* n_gt, int32_t Q, int32_t G, double* ap,
                   double* iou_r1, double* iou_r5, uint8_t* kept, void* stream);
int univtg_eval_hl(const double* sal, const int32_t* n_sal, const uint16_t* labels, const int32_t* n_clips, int32_t Q, int32_t S,
                   int32_t C, double* scratch, double* ap, double* hit, void* stream);

/* Per-(video, annotator) AP of the reference's TVSum / YouTube highlight evaluation (main/dataset.py DatasetHL.evaluate), IEEE
 * double, equal to the reference's Python floats bit for bit; univtg_b200/metrics.py evaluate_hl packs and averages.
 *   scores [V,S] f32: row v holds the n_score[v] (0..S, S <= 4096) scores the reference argsorts, ranked as torch.argsort(
 *   descending=True) on the CPU ranks them (libstdc++ std::sort, ties included).  labels [V,C,A] f32: n_label[v] (n_score[v]..C,
 *   C <= 4096) rows of A (1..32) annotator columns; a clip is positive for annotator a when its label is > the lower median of
 *   column a (median = 1, TVSum) or > 0 (median = 0, YouTube).  ap [V,A] = the reference's AP recursion over the first n_cut[v]
 *   (0..n_score[v]) ranked clips, 0 when none of them is positive. */
int univtg_eval_hl_topk(const float* scores, const int32_t* n_score, const int32_t* n_cut, const float* labels,
                        const int32_t* n_label, int32_t V, int32_t S, int32_t C, int32_t A, int32_t median, double* ap,
                        void* stream);
/* Maximum-weight bipartite matching of QFVS semantic evaluation (eval/qfvs.py calculate_semantic_matching), one per query.
 * Query q matches the machine-summary shots a[a_off[q] .. a_off[q+1]) with the ground-truth shots b[b_off[q] .. b_off[q+1]),
 * each a 64-bit mask of its tags (1..max_side per side, max_side <= 1024); the weight of a pair is popcount(x & y) /
 * popcount(x | y) (0 when both are empty).  s [Q] f64 = the total weight of a maximum-weight matching (Hungarian method, fp64
 * potentials).  The sides are read from the offsets on the device; a query with an empty side or a side longer than max_side
 * gets s = NaN, so the caller passes the largest side it packed. */
int univtg_qfvs_match(const uint64_t* a, const int32_t* a_off, const uint64_t* b, const int32_t* b_off, int32_t Q,
                      int32_t max_side, double* s, void* stream);
/* Selection step of the QFVS evaluation epoch (main/inference_qfvs.py eval_epoch) for F queries of one video, query f writing
 * slot q0 + f of the pools.  The model outputs of the three query variants (concept 1, concept 2, both) are [F, N] f32 each,
 * N = S*Lf, query f's S segments in rows f*S .. f*S+S-1.  pos [n]: the first n kept positions of mask_GT in row-major order
 * (1 <= n <= min(N, 8192)).  Per kept position i the variant score is logits (mode 0), sal (mode 1) or (0 + logits) + sal
 * (mode 2), and score[q, i] = score_both, or (score_both + score_1) + score_2 with gather = 1, in fp32.  top[q, 0..k) = the
 * indices of score.topk(k) as torch.topk on CUDA returns them (descending, NaN first; equal scores by ascending index when
 * k > 32, in the order of torch's unstable 32-wide bitonic sort of its selection when k <= 32; 1 <= k
 * <= n), a[q, 0..k) = tags[top[q, j]] (the machine side of univtg_qfvs_match, offsets q*k).  Variants 1 and 2 are read only
 * with gather = 1; logits only for modes 0 and 2, sal only for modes 1 and 2. */
int univtg_qfvs_eval_select(const float* logits1, const float* sal1, const float* logits2, const float* sal2, const float* logits_o,
                            const float* sal_o, const int32_t* pos, const uint64_t* tags, int32_t F, int32_t N, int32_t n, int32_t k,
                            int32_t mode, int32_t gather, int32_t q0, float* score, int32_t* top, uint64_t* a, void* stream);

/* LayerNorm rows: in [rows,d] f32 -> out32 [rows,d] f32 and/or out16 [rows,ld16] 16-bit (zero padded). */
int univtg_op_layernorm(const float* in, int32_t rows, int32_t d, const float* gamma, const float* beta, float eps,
                        int32_t fmt, float* out32, void* out16, int32_t ld16, void* stream);
/* Attention core.  qkv: [B*L, 3d] 16-bit, column blocks Q | K | V (heads are dh-wide sub-blocks), d = H*dh; scores are
 * scaled by 1/sqrt(dh); key_mask [B,L] f32 (1 = valid key); out [B*L,d] 16-bit; lse [B,H,L] f32 or NULL.
 * impl: 0 = tensor cores (wgmma, dh in {64,128}), 1 = SIMT (any dh). */
int univtg_op_attention(const void* qkv, const float* key_mask, void* out, float* lse, int32_t B, int32_t L, int32_t H,
                        int32_t dh, int32_t fmt, int32_t impl, void* stream);

/* LayerNorm forward with the fused store epilogue of univtg_forward (one entry per LnArgs field of csrc/rowops.h):
 *   v = (in or in16) + add16 (sum_out = v, fp32 [rows, d]);  y = (v - mean) * rstd * gamma + beta, rstd = 1/sqrt(var + eps);
 *   out32 = y;  y' = y * (mul32 or the in-kernel dropout of (rng, mask_index), as univtg_dropout_mask reads it back);
 *   out16 = 16-bit(y') [rows, ld16] (columns [d, ld16) zeroed);  out16p = 16-bit(y' + pos[b*Lv + l]) on video rows l < Lv,
 *   16-bit(y' + pos_txt[b*(L-Lv) + l - Lv]) on text rows when pos_txt is given, else 16-bit(y');  outc = 16-bit(y') at row
 *   1 + b*(Lv+1) + l of the conv-head layout for video rows;  mean_out / rstd_out [rows].  Row r = b*L + l (L = 0: unstructured).
 * fmt 0 fp16, 1 bf16, 2 fp16x3 (no dropout): add16, out16, out16p and outc are hi planes whose lo planes lie `lo` elements after
 * them.  fp32 pointers must be 16-byte and 16-bit pointers 8-byte aligned. */
typedef struct univtg_ln_fwd {
  const float* in;
  const void* in16;
  int32_t in_fmt, ld_in;
  const void* add16;
  int32_t ld_add16;
  float* sum_out;
  int32_t rows, d;
  const float* gamma;
  const float* beta;
  float eps;
  int32_t fmt;
  int64_t lo;
  int32_t L, Lv;
  float* out32;
  void* out16;
  void* out16p;
  int32_t ld16;
  const float* pos;
  const float* pos_txt;
  void* outc;
  const float* mul32;
  float* mean_out;
  float* rstd_out;
} univtg_ln_fwd;
/* kernel_used (optional) receives the instantiation that ran: 0/1/2 warp-per-row d = 1024/512/256, 3/4/5 the same with pos_txt,
 * 6/7 row-per-block d <= 1024 / <= 3072, 8/9 the same with pos_txt, 10 the 64-bit-load projector kernel (even d in (1024, 3072],
 * out16 only), 11 any d; + 12 for fp16x3. */
int univtg_op_layernorm_fwd(const univtg_ln_fwd* args, const univtg_rng* rng, int32_t mask_index, int32_t* kernel_used, void* stream);

/* Learned text positions of univtg_plan_set_txt_pos, one text row r = b*Lt + l at a time: pos[r] = drop(LayerNorm(xt[r] + table[l]))
 * (eps 1e-5; mul32, else the dropout of (rng, mask_index)); row b*L + Lv + l of xpos16 [B*L, d] = 16-bit(xt[r] + pos[r]), no other
 * row is written; mean_out / rstd_out [B*Lt] (both or neither).  d % 64 == 0, d <= 1024.  fmt 2: fp16x3, xpos16's lo plane `lo`
 * elements after it. */
typedef struct univtg_txt_pos_fwd {
  const float* xt;
  const float* table;
  const float* gamma;
  const float* beta;
  const float* mul32;
  float* pos;
  float* mean_out;
  float* rstd_out;
  void* xpos16;
  int32_t B, Lt, L, Lv, d, fmt;
  int64_t lo;
} univtg_txt_pos_fwd;
int univtg_op_txt_pos(const univtg_txt_pos_fwd* args, const univtg_rng* rng, int32_t mask_index, void* stream);

/* Sine position table of univtg_forward: c = cumsum_l(vid_mask[b]); pos[b*Lv + l, 2k + {0,1}] = {sin, cos}(c_l / (c_last + 1e-6)
 * * 2pi / dim_t[2k]) (fp32 [B*Lv, d], d even, 8-byte aligned); key_mask (optional) [B, Lv+Lt] = cat(vid_mask, txt_mask);
 * dp_out (optional) [n_sites, B] = the DropPath scales of rng (univtg_droppath_scales).  Lv <= 12288. */
int univtg_op_sine_pos(const float* vid_mask, const float* txt_mask, const float* dim_t, float* pos, float* key_mask, int32_t B, int32_t Lv,
                       int32_t Lt, int32_t d, const univtg_rng* rng, int32_t n_sites, float* dp_out, void* stream);

/* WeightedPool + cosine saliency of univtg_forward: logits [B, Lt] = x_txt . w + (1 - txt_mask) * -1e30 (scratch, written);
 * alpha = softmax_l(logits) (alpha_out optional); pooled [B, d] = sum_l alpha_l x_txt[b, l];
 * saliency [B, Lv] = x_vid . pooled / (max(|x_vid|, 1e-8) max(|pooled|, 1e-8)) + log(vid_mask + 1e-45).
 * d % 4 == 0, fp32 arrays 16-byte aligned, Lt <= 12288. */
int univtg_op_pool_saliency(const float* x_txt, const float* x_vid, const float* txt_mask, const float* vid_mask, const float* w,
                            float* pooled, float* saliency, float* alpha_out, float* logits, int32_t B, int32_t Lt, int32_t Lv, int32_t d,
                            void* stream);

/* Last conv layer of both heads: h_cls / h_span 16-bit [B*(Lv+1)+2, d] in the conv-head layout (rows 0, B*(Lv+1)+1 and the separator
 * rows zero); w_cls [3][d], w_span [2][3][d] fp32 (w[o][t][c] = W[o, c, t]); pred_logits [B*Lv] = sigmoid(z_cls), pred_spans [B*Lv, 2]
 * = (-sigmoid(z_0), sigmoid(z_1)) with z = sum_t h[row + t - 1] . w[t] + bias.  d even; fmt 2 (fp16x3): lo planes directly after the
 * hi planes ((B*(Lv+1)+2) * d elements later). */
int univtg_op_conv_head_final(const void* h_cls, const void* h_span, const float* w_cls, const float* w_span, const float* b_cls,
                              const float* b_span, float* pred_logits, float* pred_spans, int32_t B, int32_t Lv, int32_t d, int32_t fmt,
                              void* stream);

/* Attention forward with every option of the kernels: qkv, key_mask, out, lse as univtg_op_attention; causal = 1: query i sees keys
 * j <= i only (dh 64, fmt 0/1, tensor cores, no dropout); impl 0 tensor cores (dh 64 / 128), 1 SIMT (any dh); p > 0: attention
 * dropout of encoder layer `layer` of rng (univtg_attention_dropout_mask reads it back; fmt 0/1).  kernel_used (optional):
 * 0..7 tensor cores = 4 (dh 128) + 2 (bf16) + dropout, 8/9 causal fp16/bf16, 10/11 fp16x3 dh 64/128, 12/13/14 SIMT plain/dropout/fp16x3. */
typedef struct univtg_attn_fwd {
  const void* qkv;
  const float* key_mask;
  void* out;
  float* lse;
  int32_t B, L, H, dh, fmt, impl, causal;
} univtg_attn_fwd;
int univtg_op_attention_fwd(const univtg_attn_fwd* args, const univtg_rng* rng, float p, int32_t layer, int32_t* kernel_used, void* stream);

/* Attention core backward.  qkv as above; dO [B*L,d] 16-bit gradient of `out`; O = forward output (16-bit, fmt_act);
 * (same 16-bit format as qkv); lse from the forward; delta_ws [B,H,L] f32 scratch; dqkv32 [B*L,3d] f32 receives
 * dQ | dK | dV.  impl: 0 tensor cores (wgmma), 1 SIMT. */
int univtg_op_attention_bwd(const void* qkv, const void* dO, const void* O, const float* key_mask, const float* lse,
                            float* delta_ws, float* dqkv32, int32_t B, int32_t L, int32_t H, int32_t dh, int32_t fmt_act,
                            int32_t impl, void* stream);

/* delta [B, H, L] f32 = rowsum over each head's dh channels of dO o O (dO, O 16-bit [B*L, H*dh], formats fmt_do / fmt_o 0/1).
 * vec_used (optional): 1 when the 128-bit vector path ran (dh a power-of-two multiple of 8 up to 256, 16-byte aligned dO and O),
 * 0 for the scalar path. */
int univtg_op_attn_delta(const void* dO, int32_t fmt_do, const void* O, int32_t fmt_o, float* delta, int32_t B, int32_t L, int32_t H,
                         int32_t dh, int32_t* vec_used, void* stream);

/* Attention core backward with every option of the kernels, routed as univtg_backward routes it.  qkv [B*L, 3d] and dO [B*L, d]
 * 16-bit (fmt 0/1, 16-byte aligned); key_mask [B, L]; lse and delta [B, H, L] f32 (delta = univtg_op_attn_delta); dqkv32 [B*L, 3d]
 * f32; dqkv16 (optional, impl 0 and L <= 128) [B*L, 3d] 16-bit.  impl 0 tensor cores (dh 64 / 128), 1 SIMT (any dh, L up to the
 * device's opt-in shared memory / 32 bytes).  p > 0: the attention dropout of encoder layer `layer` of rng, as the forward drew it.
 * kernel_used (optional): 4 (dh 128) + 2 (bf16) + dropout = 0..7 tensor cores, 8 + dropout SIMT.  dq_mode (optional): 0 dQ | dK | dV
 * written to dqkv16 (dqkv32 untouched), 1 written to dqkv32 with dQ stored (one key tile), 2 dqkv32 zeroed and dQ accumulated
 * atomically (several key tiles, or SIMT). */
typedef struct univtg_attn_bwd {
  const void* qkv;
  const void* dO;
  const float* key_mask;
  const float* lse;
  const float* delta;
  float* dqkv32;
  void* dqkv16;
  int32_t B, L, H, dh, fmt, impl;
} univtg_attn_bwd;
int univtg_op_attention_bwd_full(const univtg_attn_bwd* args, const univtg_rng* rng, float p, int32_t layer, int32_t* kernel_used,
                                 int32_t* dq_mode, void* stream);

/* ---- CLIP feature extraction (inference only): the ViT image tower and the text tower of OpenAI CLIP
 * (reference run_on_video/clip/model.py: VisualTransformer 202-236, encode_text 339-352), which produce the video and query
 * features the grounding model consumes.  Every head is 64 wide (heads = width / 64, model.py:268); LayerNorm eps 1e-5. ---- */
typedef struct univtg_clip_config {
  int32_t embed_dim;         /* text_projection.shape[1] = visual.proj.shape[1]; multiple of 16 */
  int32_t vision_width;      /* visual.conv1.weight.shape[0]; multiple of 64, <= 1024 */
  int32_t vision_layers;     /* visual.transformer.resblocks.* count, 1..64 */
  int32_t patch_size;        /* visual.conv1.weight.shape[-1] (P) */
  int32_t image_resolution;  /* R = P * grid; frames are R x R */
  int32_t text_width;        /* ln_final.weight.shape[0]; multiple of 64, <= 1024 */
  int32_t text_layers;       /* transformer.resblocks.* count, 1..64 */
  int32_t context_length;    /* positional_embedding.shape[0]; tokens are [n, context_length] */
  int32_t vocab_size;        /* token_embedding.weight.shape[0] */
  int32_t operand_format;    /* 0 fp16, 1 bf16 GEMM / attention operands (fp32 accumulation, LayerNorm and residual stream);
                              * 2 (fp16x3) is refused */
} univtg_clip_config;
/* Number of parameter tensors univtg_clip_pack_weights expects, in this order (reference state_dict names):
 *   visual.{conv1.weight, class_embedding, positional_embedding, ln_pre.weight, ln_pre.bias},
 *   for l < vision_layers: visual.transformer.resblocks.l.{attn.in_proj_weight, attn.in_proj_bias, attn.out_proj.weight,
 *        attn.out_proj.bias, ln_1.weight, ln_1.bias, mlp.c_fc.weight, mlp.c_fc.bias, mlp.c_proj.weight, mlp.c_proj.bias,
 *        ln_2.weight, ln_2.bias},
 *   visual.{ln_post.weight, ln_post.bias, proj},
 *   token_embedding.weight, positional_embedding, for l < text_layers: transformer.resblocks.l.{same twelve},
 *   ln_final.weight, ln_final.bias, text_projection */
int univtg_clip_num_params(const univtg_clip_config* cfg);
size_t univtg_clip_packed_bytes(const univtg_clip_config* cfg);
/* params: HOST array of device pointers, contiguous tensors of element type src_dtype (0 f32, 1 fp16: released CLIP checkpoints
 * are mostly fp16).  Matrices become 16-bit GEMM operands; visual.proj and text_projection are stored transposed. */
int univtg_clip_pack_weights(const univtg_clip_config* cfg, const void* const* params, int32_t n_params, int32_t src_dtype,
                             void* packed, void* stream);
/* Workspace bytes for encoding up to n_images frames and up to n_texts token rows of text_len positions (either count may be 0).
 * The two towers share one workspace: calls on one stream may reuse it. */
size_t univtg_clip_workspace_bytes(const univtg_clip_config* cfg, int32_t n_images, int32_t n_texts, int32_t text_len);
/* encode_image of n frames -> out [n, embed_dim] f32.
 *   pixel_kind 0: uint8 [n, R, R, 3] RGB (ffmpeg rgb24); normalised in-kernel as run_on_video/preprocessing.py does:
 *                 (x / 255 - mean[c]) / (std[c] + 1e-8) with CLIP's mean and std.
 *   pixel_kind 1: f32 [n, 3, R, R], already normalised (encode_image's own input).
 * n (frames here, token rows in univtg_clip_encode_text) is at most 65535 per call. */
int univtg_clip_encode_image(const univtg_clip_config* cfg, const void* packed, const void* pixels, int32_t pixel_kind, int32_t n,
                             void* ws, size_t ws_bytes, float* out, void* stream);
/* encode_text of n token rows: tokens [n, context_length] int64 (clip.tokenize ids).  Only positions < ctx_used are computed:
 * the causal mask makes them independent of later tokens, so ctx_used = context_length is the reference's encode_text and a
 * smaller ctx_used that still covers every row's argmax (EOT) gives the same rows.  last_hidden (nullable): [n, ctx_used, text_width]
 * f32 = ln_final(x); pooled (nullable): [n, embed_dim] f32 = ln_final(x)[argmax(tokens)] @ text_projection.  The tokens are read
 * back to the host and checked before anything launches (ids in [0, vocab_size), argmax < ctx_used): the call synchronises
 * `stream` once. */
int univtg_clip_encode_text(const univtg_clip_config* cfg, const void* packed, const int64_t* tokens, int32_t n, int32_t ctx_used,
                            void* ws, size_t ws_bytes, float* last_hidden, float* pooled, void* stream);
/* Kernels one call launches: tower 0 = univtg_clip_encode_image, 1 = univtg_clip_encode_text with text_outputs bit 0 = last_hidden,
 * bit 1 = pooled. */
int univtg_clip_num_launches(const univtg_clip_config* cfg, int32_t tower, int32_t text_outputs);

/* ---- CLIP-teacher pseudo labels (reference teacher/clip2label.py): per video the top-k classes by the sum over clips of the
 * clip-class cosines (ties to the lower class index), and per chosen class the curve float32(cos) // th with the runs of its
 * maximum that end before the last clip.  Cosines use a / max(||a||, 1e-8) and are computed in fp64 from the f32 features.
 * cls: [C, D] f32 class features, D <= 1024. ---- */
size_t univtg_teacher_class_bytes(int32_t C, int32_t D);
/* Normalised class table (fp16x3 planes and fp64 norms) into cls_ws (univtg_teacher_class_bytes); kept for every later call. */
int univtg_teacher_prepare_classes(const float* cls, int32_t C, int32_t D, void* cls_ws, void* stream);
/* Workspace for one univtg_teacher_label call of V videos with S clips in total (includes a [V, C rounded up to 16] f32 matrix). */
size_t univtg_teacher_chunk_bytes(int32_t V, int64_t S, int32_t C, int32_t D);
/* feats [S, D] f32 (videos concatenated), offsets [V + 1] int32 on the device, every video 1..65535 clips (checked by the
 * caller); topk in 1..16, finite th >= 2^-30 (so that |bins| <= 1 / th + 1 fit in int32).
 * out: int32 [2 V topk + 2 S topk + 1], zeroed and then written as
 *   idx  [V, topk]  chosen class per rank (-1 when C < topk),
 *   nwin [V, topk]  windows per rank (0: no window, the line is skipped),
 *   win  [S, topk]  rows off_v .. off_v + nwin - 1: (first clip << 16) | last clip of each window (uint32),
 *   bins [S, topk]  float32(cos) // th of every clip (INT32_MIN stands for -0.0),
 *   and the number of videos that were rescored over every class because the approximate ranking could not be certified. */
int univtg_teacher_label(const float* cls, const void* cls_ws, int32_t C, int32_t D, const float* feats, const int32_t* offsets,
                         int32_t V, int64_t S, int32_t topk, double th, void* ws, size_t ws_bytes, int32_t* out, void* stream);
/* Host only: out[i] = x[i] // th with Python's float floor division, the function the curves use on the device. */
int univtg_debug_py_floordiv(const double* x, int64_t n, double th, double* out);

#ifdef __cplusplus
}
#endif
#endif /* UNIVTG_B200_H_ */
