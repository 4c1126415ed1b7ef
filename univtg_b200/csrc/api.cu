// C-ABI layer (include/univtg_b200.h): weight packing, plan construction (shapes and tile widths) and the forward
// orchestration of reference Model.forward (model/univtg.py:105-155), shared by inference and training.
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <new>
#include <vector>

#include "plan.h"
#include "ptx.cuh"

extern "C" {

const char* univtg_last_error(void) { return uv::last_error(); }
int univtg_abi_version(void) { return UNIVTG_ABI_VERSION; }

int univtg_num_params(const univtg_config* cfg) {
  if (!check_cfg(cfg)) return -1;
  return ParamIndex(*cfg).count();
}

size_t univtg_packed_bytes(const univtg_config* cfg) {
  if (!check_cfg(cfg)) return 0;
  return planes(*cfg) * make_layout(*cfg).total;
}

// mode 0: everything; mode 1: only the fp32 vectors / small fp32 tensors (the 16-bit matrices are kept current by univtg_adamw_step)
static int pack_impl(const univtg_config* cfg, const float* const* params, int32_t n_params, void* packed, void* stream, int mode) {
  if (!check_cfg(cfg)) return 1;
  const int expect = univtg_num_params(cfg);
  if (n_params != expect || !params || !packed) {
    set_error("univtg_pack_weights: expected %d parameter tensors, got %d", expect, n_params);
    return 1;
  }
  for (int i = 0; i < n_params; ++i)
    if (!params[i]) {
      set_error("univtg_pack_weights: parameter %d is null", i);
      return 1;
    }
  const PackedLayout L = make_layout(*cfg);
  const int d = cfg->hidden_dim, ff = cfg->dim_feedforward;
  Packer pk;
  pk.base = reinterpret_cast<uint8_t*>(packed);
  pk.fmt = kernel_fmt(*cfg);
  pk.lo = is_split(*cfg) ? (long long)L.total : 0;
  pk.st = (cudaStream_t)stream;
  pk.tab.n = 0;
  pk.skip_matrices = mode == 1;
  const ParamIndex ix(*cfg);
  const float* type_emb = params[ix.type()];  // token_type_embeddings.weight [2, d]
  for (int s = 0; s < 2; ++s) {
    const ProjPacked* pp = s == 0 ? L.vid : L.txt;
    for (int i = 0; i < cfg->n_input_proj; ++i) {
      const float* const* pr = params + (s == 0 ? ix.vid(i, 0) : ix.txt(i, 0));
      pk.vec(pr[0], pp[i].ln_w, pp[i].din);
      pk.vec(pr[1], pp[i].ln_b, pp[i].din);
      pk.rows(pr[2], pp[i].w16, d, pp[i].din, pp[i].kpad);
      const bool last = (i == cfg->n_input_proj - 1);
      // token_type_embeddings: index 1 for video tokens, 0 for text tokens (model/univtg.py:114-115)
      pk.vec(pr[3], pp[i].bias, d, last ? type_emb + (s == 0 ? d : 0) : nullptr);
    }
  }
  for (int l = 0; l < cfg->enc_layers; ++l) {
    const LayerPacked& lp = L.layer[l];
    const float* const* pr = params + ix.layer(l, 0);
    pk.rows(pr[0], lp.w_in, 3 * d, d, d);
    pk.vec(pr[1], lp.b_in, 3 * d);
    pk.rows(pr[2], lp.w_out, d, d, d);
    pk.vec(pr[3], lp.b_out, d);
    pk.rows(pr[4], lp.w1, ff, d, d);
    pk.vec(pr[5], lp.b1, ff);
    pk.rows(pr[6], lp.w2, d, ff, ff);
    pk.vec(pr[7], lp.b2, d);
    pk.vec(pr[8], lp.n1w, d);
    pk.vec(pr[9], lp.n1b, d);
    pk.vec(pr[10], lp.n2w, d);
    pk.vec(pr[11], lp.n2b, d);
  }
  // span_embed.layers.{0,1,2}, class_embed.layers.{0,1,2}
  const float* const* sp = params + ix.span(0);
  const float* const* cl = params + ix.cls(0);
  // fused first conv: rows [0,d) = class_embed.layers.0, rows [d,2d) = span_embed.layers.0
  pk.conv(cl[0], L.conv1_w, d, d);
  pk.conv(sp[0], L.conv1_w + (size_t)d * 3 * d * 2, d, d);
  pk.vec(cl[1], L.conv1_b, d);
  pk.vec(sp[1], L.conv1_b + (size_t)d * 4, d);
  pk.conv(cl[2], L.conv2c_w, d, d);
  pk.vec(cl[3], L.conv2c_b, d);
  pk.conv(sp[2], L.conv2s_w, d, d);
  pk.vec(sp[3], L.conv2s_b, d);
  pk.conv_f32(cl[4], L.conv3c_w, 1, d);
  pk.vec(cl[5], L.conv3c_b, 1);
  pk.conv_f32(sp[4], L.conv3s_w, 2, d);
  pk.vec(sp[5], L.conv3s_b, 2);
  pk.vec(params[ix.pool()], L.pool_w, d);
  pk.flush();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("univtg_pack_weights: %s", cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

int univtg_pack_weights(const univtg_config* cfg, const float* const* params, int32_t n_params, void* packed, void* stream) {
  return pack_impl(cfg, params, n_params, packed, stream, 0);
}
int univtg_pack_vectors(const univtg_config* cfg, const float* const* params, int32_t n_params, void* packed, void* stream) {
  return pack_impl(cfg, params, n_params, packed, stream, 1);
}

// Segments of the flat parameter buffer (univtg_pack_weights order, every tensor padded to a multiple of 4 floats) that are GEMM
// weight matrices, with their place in `packed`.
static int make_pack_segments(const univtg_config& c, void* packed, PackSegTable& t) {
  const PackedLayout L = make_layout(c);
  uint8_t* base = reinterpret_cast<uint8_t*>(packed);
  const long long d = c.hidden_dim, ff = c.dim_feedforward;
  t.n = 0;
  t.fmt = c.operand_format;
  long long off = 0;  // floats
  auto skip = [&](long long numel) { off += (numel + 3) / 4 * 4; };
  auto seg = [&](long long numel, size_t dst, int kind, int rows, int cols, int ld) {
    if (t.n >= kMaxPackSegs) return 1;
    PackSeg& s = t.s[t.n++];
    s.start4 = off / 4;
    s.end4 = (off + numel + 3) / 4;
    s.dst = base + dst;
    s.kind = kind;
    s.rows = rows;
    s.cols = cols;
    s.ld = ld;
    skip(numel);
    return 0;
  };
  int rc = 0;
  for (int sdx = 0; sdx < 2; ++sdx) {
    const ProjPacked* pp = sdx == 0 ? L.vid : L.txt;
    for (int i = 0; i < c.n_input_proj; ++i) {
      skip(pp[i].din);
      skip(pp[i].din);
      rc |= seg(d * pp[i].din, pp[i].w16, 0, (int)d, pp[i].din, pp[i].kpad);
      skip(d);
    }
  }
  skip(2 * d);  // token_type_embeddings
  for (int l = 0; l < c.enc_layers; ++l) {
    const LayerPacked& lp = L.layer[l];
    rc |= seg(3 * d * d, lp.w_in, 0, (int)(3 * d), (int)d, (int)d);
    skip(3 * d);
    rc |= seg(d * d, lp.w_out, 0, (int)d, (int)d, (int)d);
    skip(d);
    rc |= seg(ff * d, lp.w1, 0, (int)ff, (int)d, (int)d);
    skip(ff);
    rc |= seg(d * ff, lp.w2, 0, (int)d, (int)ff, (int)ff);
    skip(d);
    skip(d); skip(d); skip(d); skip(d);
  }
  // span_embed.layers.{0,1,2} then class_embed.layers.{0,1,2}; fused first conv: rows [0,d) class, [d,2d) span
  rc |= seg(d * d * 3, L.conv1_w + (size_t)d * 3 * d * 2, 1, (int)d, (int)d, 0);
  skip(d);
  rc |= seg(d * d * 3, L.conv2s_w, 1, (int)d, (int)d, 0);
  skip(d);
  skip(2 * d * 3);
  skip(2);
  rc |= seg(d * d * 3, L.conv1_w, 1, (int)d, (int)d, 0);
  skip(d);
  rc |= seg(d * d * 3, L.conv2c_w, 1, (int)d, (int)d, 0);
  skip(d);
  skip(1 * d * 3);
  skip(1);
  skip(d);  // weightedpool.weight
  if (rc) {
    set_error("univtg_adamw_step: too many weight matrices for the pack-segment table");
    return -1;
  }
  return (int)(off);  // total floats of the flat buffer
}

int univtg_adamw_step(float* params, float* grads, float* exp_avg, float* exp_avg_sq, size_t n, float lr, float beta1, float beta2,
                      float eps, float weight_decay, int32_t step, float max_grad_norm, int32_t write_clipped_grads,
                      float* scratch3, const univtg_config* cfg, void* packed, void* stream) {
  if (cfg == nullptr || packed == nullptr)
    return uv::adamw_step_impl(params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, max_grad_norm,
                               write_clipped_grads, scratch3, nullptr, stream);
  if (!check_cfg(cfg) || refuse_split(*cfg, "univtg_adamw_step")) return 1;
  PackSegTable t;
  const int total = make_pack_segments(*cfg, packed, t);
  if (total < 0) return 1;
  if ((size_t)total > n) {
    set_error("univtg_adamw_step: flat buffer has %zu floats, the config's parameters need %d", n, total);
    return 1;
  }
  return uv::adamw_step_impl(params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, max_grad_norm,
                             write_clipped_grads, scratch3, &t, stream);
}

int univtg_adamw_step_dev(float* params, float* grads, float* exp_avg, float* exp_avg_sq, size_t n, const float* lr_dev,
                          float beta1, float beta2, float eps, float weight_decay, int32_t* step_dev, float max_grad_norm,
                          int32_t write_clipped_grads, float* scratch3, const univtg_config* cfg, void* packed,
                          const float* bc_table, int32_t table_len, void* stream) {
  const char* fn = "univtg_adamw_step_dev";
  UV_REQ(params && grads && exp_avg && exp_avg_sq && scratch3, "%s: null params, grads, exp_avg, exp_avg_sq or scratch3", fn);
  UV_REQ(lr_dev && step_dev && bc_table, "%s: null lr_dev, step_dev or bc_table", fn);
  UV_REQ(n % 4 == 0, "%s: n %zu must be a multiple of 4", fn, n);
  UV_REQ(table_len >= 1, "%s: table_len %d must be >= 1", fn, (int)table_len);
  UV_REQ(al_(params, 16) && al_(grads, 16) && al_(exp_avg, 16) && al_(exp_avg_sq, 16), "%s: flat buffers must be 16-byte aligned", fn);
  UV_REQ(al_(lr_dev, 4) && al_(step_dev, 4) && al_(bc_table, 4) && al_(scratch3, 4), "%s: misaligned lr_dev, step_dev, bc_table or scratch3", fn);
  UV_REQ((cfg == nullptr) == (packed == nullptr), "%s: cfg and packed must both be given or both be NULL", fn);
  uv::AdamDevState dev{lr_dev, step_dev, bc_table, table_len};
  if (cfg == nullptr)
    return uv::adamw_step_impl(params, grads, exp_avg, exp_avg_sq, n, 0.f, beta1, beta2, eps, weight_decay, 1, max_grad_norm,
                               write_clipped_grads, scratch3, nullptr, stream, &dev);
  if (!check_cfg(cfg) || refuse_split(*cfg, fn)) return 1;
  PackSegTable t;
  const int total = make_pack_segments(*cfg, packed, t);
  if (total < 0) return 1;
  UV_REQ((size_t)total <= n, "%s: flat buffer has %zu floats, the config's parameters need %d", fn, n, total);
  return uv::adamw_step_impl(params, grads, exp_avg, exp_avg_sq, n, 0.f, beta1, beta2, eps, weight_decay, 1, max_grad_norm,
                             write_clipped_grads, scratch3, &t, stream, &dev);
}

int univtg_adamw_bias_table(float beta1, float beta2, int32_t len, float* out_host) {
  const char* fn = "univtg_adamw_bias_table";
  UV_REQ(out_host != nullptr, "%s: null out_host", fn);
  UV_REQ(len >= 1, "%s: len %d must be >= 1", fn, (int)len);
  UV_REQ(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f, "%s: betas (%g, %g) must be in [0, 1)", fn, (double)beta1,
         (double)beta2);
  for (int32_t t = 1; t <= len; ++t) uv::adamw_bias_row(beta1, beta2, t, out_host + 2 * (size_t)(t - 1), out_host + 2 * (size_t)(t - 1) + 1);
  return 0;
}

int32_t univtg_adamw_bias_table_len(float beta1, float beta2) {
  if (!(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f)) {
    set_error("univtg_adamw_bias_table_len: betas (%g, %g) must be in [0, 1)", (double)beta1, (double)beta2);
    return 0;
  }
  // both terms are non-decreasing in t (pow of a base in [0, 1) falls, and the float rounding is monotone): the first t where
  // both are 1.0f is where the table may end
  for (int32_t t = 1; t <= (1 << 26); ++t) {
    float b1, b2;
    uv::adamw_bias_row(beta1, beta2, t, &b1, &b2);
    if (b1 == 1.f && b2 == 1.f) return t;
  }
  set_error("univtg_adamw_bias_table_len: the bias corrections of betas (%g, %g) do not reach 1.0f within 2^26 steps", (double)beta1,
            (double)beta2);
  return 0;
}

}  // extern "C"

extern "C" {

size_t univtg_workspace_bytes(const univtg_config* cfg, const univtg_shape* shape) {
  if (!check_cfg(cfg) || !check_shape(shape)) return 0;
  return planes(*cfg) * make_infer_ws(*cfg, *shape, make_layout(*cfg), nullptr).total;
}

int univtg_plan_create(const univtg_config* cfg, const univtg_shape* shape, const void* packed, void* workspace,
                       const float* dim_t, void* stream, univtg_plan** out) {
  if (!check_cfg(cfg) || !check_shape(shape)) return 1;
  if (!packed || !workspace || !dim_t || !out) {
    set_error("univtg_plan_create: null argument");
    return 1;
  }
  univtg_plan* P = new (std::nothrow) univtg_plan;
  if (!P) {
    set_error("out of host memory");
    return 1;
  }
  memset(static_cast<void*>(P), 0, sizeof(*P));
  P->cfg = *cfg;
  P->shp = *shape;
  P->lay = make_layout(*cfg);
  P->packed = reinterpret_cast<const uint8_t*>(packed);
  P->ws = reinterpret_cast<uint8_t*>(workspace);
  P->dim_t = dim_t;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&P->num_sms, cudaDevAttrMultiProcessorCount, dev);
  if (P->num_sms <= 0) P->num_sms = 132;
  const int d = cfg->hidden_dim, ff = cfg->dim_feedforward;
  P->B = shape->batch;
  P->Lv = shape->l_vid;
  P->Lt = shape->l_txt;
  P->L = P->Lv + P->Lt;
  P->d = d;
  P->ff = ff;
  P->H = cfg->nheads;
  P->dh = d / cfg->nheads;
  P->M = P->B * P->L;
  P->Mv = P->B * P->Lv;
  P->Mt = P->B * P->Lt;
  P->Mh = P->B * (P->Lv + 1);
  if (is_split(*cfg)) {
    P->pk_lo = (long long)(P->lay.total / 2);
    P->ws_lo = (long long)(make_infer_ws(*cfg, *shape, P->lay, nullptr).total / 2);
  }
  if (univtg_prepare_workspace(cfg, shape, workspace, 0, stream) != 0) {  // zero rows of the conv-head buffers
    delete P;
    return 1;
  }
  // per-launch tile widths: fill the SMs with as little wave quantisation as possible (fp16x3 walks every K three times)
  const int sms = P->num_sms, M = P->M, Mh = P->Mh, kx = is_split(*cfg) ? 3 : 1;
  for (int i = 0; i < cfg->n_input_proj; ++i)
    P->bn_proj[i] = tile_for(sms, 16, MNK{P->Mv, d, kx * P->lay.vid[i].kpad}, MNK{P->Mt, d, kx * P->lay.txt[i].kpad}).bn;
  P->bn_qkv = tile_for(sms, 16, MNK{M, 2 * d, kx * d}, MNK{M, d, kx * d}).bn;
  P->bn_out = tile_for(sms, 16, MNK{M, d, kx * d}).bn;
  P->bn_ffn1 = tile_for(sms, 16, MNK{M, ff, kx * d}).bn;
  P->bn_ffn2 = tile_for(sms, 16, MNK{M, d, kx * ff}).bn;
  P->bn_conv1 = tile_for(sms, 16, MNK{Mh, 2 * d, kx * 3 * d}).bn;
  P->bn_conv2 = tile_for(sms, 16, MNK{Mh, d, kx * 3 * d}, MNK{Mh, d, kx * 3 * d}).bn;
  P->launches = 1 + 3 * cfg->n_input_proj + 7 * cfg->enc_layers + 6;
  *out = P;
  return 0;
}

void univtg_plan_destroy(univtg_plan* plan) {
  if (!plan) return;
  for (int i = 0; i < kMaxMarks; ++i)
    if (plan->marks[i]) cudaEventDestroy(plan->marks[i]);
  delete plan;
}

int univtg_plan_set_input_format(univtg_plan* plan, int32_t fmt) {
  if (!plan || fmt < 0 || fmt > 2) {
    set_error("univtg_plan_set_input_format: format must be 0 (f32), 1 (fp16) or 2 (bf16)");
    return 1;
  }
  plan->in_fmt = fmt;
  return 0;
}

int univtg_plan_set_attention_dropout(univtg_plan* plan, float p) {
  if (!plan || !(p >= 0.f && p < 1.f)) {
    set_error("univtg_plan_set_attention_dropout: p must be in [0, 1), got %g", (double)p);
    return 1;
  }
  plan->attn_dropout = p;
  return 0;
}

int univtg_plan_set_seed_source(univtg_plan* plan, const uint64_t* seed_dev) {
  UV_REQ(plan != nullptr, "univtg_plan_set_seed_source: null plan");
  UV_REQ(al_(seed_dev, 8), "univtg_plan_set_seed_source: seed_dev must be 8-byte aligned");
  plan->seed_dev = reinterpret_cast<const unsigned long long*>(seed_dev);
  return 0;
}

int univtg_plan_set_txt_pos(univtg_plan* plan, const univtg_txt_pos* tp) {
  if (!plan) {
    set_error("univtg_plan_set_txt_pos: null plan");
    return 1;
  }
  if (tp == nullptr) {
    plan->txt_pos_on = 0;
    memset(&plan->txt_pos, 0, sizeof(plan->txt_pos));
    return 0;
  }
  if (!tp->table || !tp->ln_weight || !tp->ln_bias || !tp->scratch) {
    set_error("univtg_plan_set_txt_pos: null table, LayerNorm term or scratch");
    return 1;
  }
  if (plan->Lt > tp->max_q_l) {
    set_error("univtg_plan_set_txt_pos: %d text tokens but the position table has max_q_l = %d rows", plan->Lt, tp->max_q_l);
    return 1;
  }
  if (plan->d % 64 != 0 || plan->d > 1024) {
    set_error("univtg_plan_set_txt_pos: hidden_dim %d must be a multiple of 64 and <= 1024", plan->d);
    return 1;
  }
  plan->txt_pos = *tp;
  plan->txt_pos_on = 1;
  return 0;
}

size_t univtg_txt_pos_scratch_bytes(const univtg_config* cfg, const univtg_shape* shape) {
  if (!check_cfg(cfg) || !check_shape(shape)) return 0;
  return make_txt_pos_ws(*cfg, *shape, nullptr).total;
}

int univtg_plan_set_profiling(univtg_plan* plan, int32_t enable) {
  if (!plan) return 1;
  plan->profiling = enable ? 1 : 0;
  plan->n_marks = 0;
  return 0;
}

int univtg_plan_read_profile(univtg_plan* plan, float* ms, int32_t* kinds, int32_t cap) {
  if (!plan || !ms || !kinds) return -1;
  if (plan->n_marks < 2) return 0;
  cudaError_t e = cudaEventSynchronize(plan->marks[plan->n_marks - 1]);
  if (e != cudaSuccess) {
    set_error("profile sync: %s", cudaGetErrorString(e));
    return -1;
  }
  int n = 0;
  for (int i = 1; i < plan->n_marks && n < cap; ++i, ++n) {
    cudaEventElapsedTime(&ms[n], plan->marks[i - 1], plan->marks[i]);
    kinds[n] = plan->mark_kind[i];
  }
  return n;
}

int univtg_forward_num_launches(const univtg_plan* plan) { return plan ? plan->launches + (plan->txt_pos_on ? 1 : 0) : -1; }
int64_t univtg_launch_count(void) { return (int64_t)*uv::launch_counter(); }

}  // extern "C"

int run_forward(univtg_plan* P, const FwdBufs& W, const float* src_txt, const float* src_txt_mask, const float* src_vid,
                const float* src_vid_mask, const float* droppath_scale, const float* const* drop_masks, const univtg_rng* rng,
                float* pred_logits, float* pred_spans, float* vid_mem_proj, float* txt_mem_proj, float* saliency_scores,
                cudaStream_t st) {
  const univtg_config& c = P->cfg;
  const PackedLayout& Lw = P->lay;
  const uint8_t* pk = P->packed;
  auto W16 = [&](size_t off) { return reinterpret_cast<const uint16_t*>(pk + off); };
  auto F32 = [&](size_t off) { return reinterpret_cast<const float*>(pk + off); };
  const int d = P->d, ff = P->ff, fmt = kernel_fmt(c), M = P->M, L = P->L, Lv = P->Lv, Lt = P->Lt, sms = P->num_sms;
  // fp16x3: element offsets of the lo planes of the packed weights and of the workspace's 16-bit buffers (0: one plane)
  const int split = is_split(c) ? 1 : 0;
  const long long pk_lo = P->pk_lo, ws_lo = P->ws_lo;
  int rc = 0;
  GemmGroup g;
  auto group = [&](int num) { reset_group(g, num, fmt, split, ws_lo); };
  // every launch is followed by a profiling mark of its kind: 0 row kernel, 1 tensor-core GEMM, 2 attention
  auto marked = [&](int r, int kind) {
    if (r == 0) prof_mark(P, st, kind);
    return r;
  };

  // train-mode randomness: explicit tensors (the caller drew them, e.g. with the reference's torch calls) win over `rng`
  const bool dp_rng = droppath_scale == nullptr && rng != nullptr && rng->droppath > 0.f;
  const bool drop_rng = drop_masks == nullptr && rng != nullptr && rng->input_dropout > 0.f;
  const bool attn_rng = rng != nullptr && P->attn_dropout > 0.f;  // attention dropout: always in-kernel, training only
  const bool training = W.mean1[0] != nullptr;
  // learned text positions: pos_t of the text rows of q = k = x + pos (zeros when off)
  const TxtPosWs TP = P->txt_pos_on ? make_txt_pos_ws(c, P->shp, P->txt_pos.scratch) : TxtPosWs{};
  prof_begin(P, st);
  rc = launch_sine_pos(src_vid_mask, src_txt_mask, P->dim_t, W.pos, W.key_mask, P->B, Lv, Lt, d, st, dp_rng ? W.dp_scale : nullptr,
                       W.dp_scale ? 2 * c.enc_layers : 0, rng ? rng->seed : 0ull, rng ? 1.0f - rng->droppath : 1.f,
                       rng ? P->seed_dev : nullptr);
  rc = marked(rc, 0);
  if (rc) return rc;
  if (dp_rng) droppath_scale = W.dp_scale;

  // ---- input projectors (LinearLayer: LN -> Dropout -> Linear -> ReLU): one grouped GEMM per depth (video + text) ----
  for (int i = 0; i < c.n_input_proj; ++i) {
    for (int s = 0; s < 2; ++s) {
      const ProjPacked& pp = s == 0 ? Lw.vid[i] : Lw.txt[i];
      LnArgs a;
      memset(&a, 0, sizeof(a));
      a.in = i == 0 ? (s == 0 ? src_vid : src_txt) : (s == 0 ? W.p_vid32[i - 1] : W.p_txt32[i - 1]);
      if (i == 0 && P->in_fmt != 0) {
        a.in16 = reinterpret_cast<const uint16_t*>(a.in);
        a.in_fmt = P->in_fmt - 1;
      }
      a.ld_in = pp.din;
      a.rows = s == 0 ? P->Mv : P->Mt;
      a.d = pp.din;
      a.gamma = F32(pp.ln_w);
      a.beta = F32(pp.ln_b);
      a.eps = 1e-5f;
      a.fmt = fmt;
      a.split = split;
      a.lo = ws_lo;
      a.out16 = s == 0 ? W.a_vid[i] : W.a_txt[i];
      a.ld16 = pp.kpad;
      a.mul32 = drop_masks ? drop_masks[s * c.n_input_proj + i] : nullptr;
      if (drop_rng) a.drop = plan_drop_spec(P, rng, (unsigned int)(s * c.n_input_proj + i), rng->input_dropout);
      a.mean_out = s == 0 ? W.pmean_v[i] : W.pmean_t[i];
      a.rstd_out = s == 0 ? W.prstd_v[i] : W.prstd_t[i];
      rc = marked(launch_layernorm(a, st), 0);
      if (rc) return rc;
    }
    group(2);
    const bool last = (i == c.n_input_proj - 1);
    const int bn = P->bn_proj[i];
    GemmProblem& pv = g.p[0];
    GemmProblem& pt = g.p[1];
    rc |= setup_linear(pv, W.a_vid[i], P->Mv, Lw.vid[i].kpad, Lw.vid[i].kpad, W16(Lw.vid[i].w16), d, Lw.vid[i].kpad, bn, ws_lo, pk_lo);
    rc |= setup_linear(pt, W.a_txt[i], P->Mt, Lw.txt[i].kpad, Lw.txt[i].kpad, W16(Lw.txt[i].w16), d, Lw.txt[i].kpad, bn, ws_lo, pk_lo);
    if (rc) return rc;
    pv.bias = F32(Lw.vid[i].bias);
    pt.bias = F32(Lw.txt[i].bias);
    if (!last) {
      pv.act = pt.act = ACT_RELU;
      pv.out32 = W.p_vid32[i];
      pt.out32 = W.p_txt32[i];
      pv.ld32 = pt.ld32 = d;
    } else {
      // video tokens -> stream rows b*L + l; text tokens -> rows b*L + Lv + l   (cat on the sequence axis, univtg.py:119)
      pv.rps_in = Lv;
      pv.rps_out = L;
      pt.rps_in = Lt;
      pt.rps_out = L;
      pt.row_off = Lv;
      pv.out32 = pt.out32 = W.x32;
      pv.ld32 = pt.ld32 = d;
      pv.out16 = pt.out16 = W.xin16[0];
      pv.out16p = pt.out16p = W.xpos16[0];
      pv.ld16 = pt.ld16 = d;
      pv.addtab = W.pos;
      pv.ld_addtab = d;
      pv.out32_id = vid_mem_proj;
      pt.out32_id = W.txtproj32;
      pv.ld32_id = pt.ld32_id = d;
    }
    rc = marked(launch_gemm_group(g, bn, sms, st), 1);
    if (rc) return rc;
  }
  if (P->txt_pos_on) {  // pos_t = Dropout(LayerNorm(x_t + P[l])); text rows of xpos16[0] := 16-bit(x_t + pos_t)
    TxtPosArgs a;
    memset(&a, 0, sizeof(a));
    a.xt = W.txtproj32;
    a.table = P->txt_pos.table;
    a.gamma = P->txt_pos.ln_weight;
    a.beta = P->txt_pos.ln_bias;
    if (training) {
      a.mul32 = P->txt_pos.drop_mul;
      if (!a.mul32 && rng != nullptr && rng->input_dropout > 0.f)
        a.drop = plan_drop_spec(P, rng, (unsigned int)(2 * c.n_input_proj), rng->input_dropout);
      a.mean_out = TP.mean;
      a.rstd_out = TP.rstd;
    }
    a.pos = TP.pos;
    a.xpos16 = W.xpos16[0];
    a.B = P->B;
    a.Lt = Lt;
    a.L = L;
    a.Lv = Lv;
    a.d = d;
    a.fmt = fmt;
    a.split = split;
    a.lo = ws_lo;
    rc = marked(launch_txt_pos(a, st), 0);
    if (rc) return rc;
  }

  // ---- encoder layers (post-norm; TransformerEncoderLayer.forward_post) ----
  for (int l = 0; l < c.enc_layers; ++l) {
    const LayerPacked& lp = Lw.layer[l];
    // q = k = x + pos -> columns [0, 2d) of qkv16; v = x -> columns [2d, 3d)   (in_proj rows: Wq, Wk, Wv)
    group(2);
    rc |= setup_linear(g.p[0], W.xpos16[l], M, d, d, W16(lp.w_in), 2 * d, d, P->bn_qkv, ws_lo, pk_lo);
    rc |= setup_linear(g.p[1], W.xin16[l], M, d, d, W16(lp.w_in) + (size_t)2 * d * d, d, d, P->bn_qkv, ws_lo, pk_lo);
    if (rc) return rc;
    g.p[0].bias = F32(lp.b_in);
    g.p[0].out16 = W.qkv16[l];
    g.p[0].ld16 = 3 * d;
    g.p[1].bias = F32(lp.b_in) + 2 * d;
    g.p[1].out16 = W.qkv16[l] + 2 * d;
    g.p[1].ld16 = 3 * d;
    rc = marked(launch_gemm_group(g, P->bn_qkv, sms, st), 1);
    if (rc) return rc;
    {
      AttnArgs a;
      memset(&a, 0, sizeof(a));
      a.key_mask = W.key_mask;
      a.out = W.attn16[l];
      a.lse = W.lse[l];
      a.scale = 1.0f / sqrtf((float)P->dh);  // torch MHA: q * dh**-0.5 before q k^T
      a.B = P->B;
      a.L = L;
      a.H = P->H;
      a.dh = P->dh;
      a.d = d;
      a.fmt = fmt;
      a.split = split;
      a.lo_qkv = a.lo_out = ws_lo;
      if (attn_rng) a.drop = plan_drop_spec(P, rng, (unsigned int)l, P->attn_dropout);
      if (P->dh == 64 || P->dh == 128) {
        if (make_tmap_op(&a.tm_qkv, W.qkv16[l], (uint64_t)M, (uint64_t)3 * d, (uint64_t)3 * d, 128, 64, ws_lo)) return 1;
        rc = launch_attention(a, st);
      } else {
        rc = launch_attention_simt(a, W.qkv16[l], st);
      }
      rc = marked(rc, 2);
      if (rc) return rc;
    }
    group(1);
    rc = setup_linear(g.p[0], W.attn16[l], M, d, d, W16(lp.w_out), d, d, P->bn_out, ws_lo, pk_lo);
    if (rc) return rc;
    g.p[0].bias = F32(lp.b_out);
    g.p[0].rps_in = L;
    g.p[0].rps_out = L;
    g.p[0].row_scale = droppath_scale ? droppath_scale + (size_t)(2 * l) * P->B : nullptr;
    g.p[0].out16 = W.br16;  // DropPath-scaled branch; the LayerNorm kernel adds it to the fp32 residual stream
    g.p[0].ld16 = d;
    rc = marked(launch_gemm_group(g, P->bn_out, sms, st), 1);
    if (rc) return rc;
    {
      LnArgs a;
      memset(&a, 0, sizeof(a));
      a.in = W.x32;
      a.ld_in = d;
      a.add16 = W.br16;
      a.ld_add16 = d;
      a.sum_out = W.y1[l];
      a.rows = M;
      a.d = d;
      a.gamma = F32(lp.n1w);
      a.beta = F32(lp.n1b);
      a.eps = 1e-5f;
      a.fmt = fmt;
      a.split = split;
      a.lo = ws_lo;
      a.out32 = W.x1_32;
      a.out16 = W.x1_16[l];
      a.ld16 = d;
      a.mean_out = W.mean1[l];
      a.rstd_out = W.rstd1[l];
      rc = marked(launch_layernorm(a, st), 0);
      if (rc) return rc;
    }
    group(1);
    rc = setup_linear(g.p[0], W.x1_16[l], M, d, d, W16(lp.w1), ff, d, P->bn_ffn1, ws_lo, pk_lo);
    if (rc) return rc;
    g.p[0].bias = F32(lp.b1);
    g.p[0].act = ACT_GELU;
    g.p[0].out16 = W.h16[l];
    g.p[0].ld16 = ff;
    if (W.dgelu16[l]) {
      g.p[0].dact16 = W.dgelu16[l];
      g.p[0].ld_dact = ff;
    }
    rc = marked(launch_gemm_group(g, P->bn_ffn1, sms, st), 1);
    if (rc) return rc;
    group(1);
    rc = setup_linear(g.p[0], W.h16[l], M, ff, ff, W16(lp.w2), d, ff, P->bn_ffn2, ws_lo, pk_lo);
    if (rc) return rc;
    g.p[0].bias = F32(lp.b2);
    g.p[0].rps_in = L;
    g.p[0].rps_out = L;
    g.p[0].row_scale = droppath_scale ? droppath_scale + (size_t)(2 * l + 1) * P->B : nullptr;
    g.p[0].out16 = W.br16;
    g.p[0].ld16 = d;
    rc = marked(launch_gemm_group(g, P->bn_ffn2, sms, st), 1);
    if (rc) return rc;
    {
      LnArgs a;
      memset(&a, 0, sizeof(a));
      a.in = W.x1_32;
      a.ld_in = d;
      a.add16 = W.br16;
      a.ld_add16 = d;
      a.sum_out = W.y2[l];
      a.rows = M;
      a.d = d;
      a.gamma = F32(lp.n2w);
      a.beta = F32(lp.n2b);
      a.eps = 1e-5f;
      a.fmt = fmt;
      a.split = split;
      a.lo = ws_lo;
      a.L = L;
      a.Lv = Lv;
      a.out32 = W.x32;
      a.out16 = W.xin16[l + 1];
      a.out16p = W.xpos16[l + 1];
      a.ld16 = d;
      a.pos = W.pos;
      a.pos_txt = TP.pos;
      a.mean_out = W.mean2[l];
      a.rstd_out = W.rstd2[l];
      if (l == c.enc_layers - 1) a.outc = W.hA;  // vid_mem = memory[:, :Lv] feeds the conv heads
      rc = marked(launch_layernorm(a, st), 0);
      if (rc) return rc;
    }
  }

  // ---- heads: conv layers (k=3, pad=1) as 3-tap GEMMs over the separated layout, then the final conv and the pooling ----
  auto conv_problem = [&](GemmProblem& p, const uint16_t* A, int lda, const uint16_t* Wc, int N, const float* bias, uint16_t* out,
                          int ldo, int bn) -> int {
    const int r = conv_fwd_problem(p, P->Mh, A, lda, d, Wc, N, bn, ws_lo, pk_lo);
    p.bias = bias;
    p.act = ACT_RELU;
    p.rps_in = Lv + 1;
    p.rps_out = Lv + 1;
    p.row_off = 1;
    p.zero_sep = 1;
    p.out16 = out;
    p.ld16 = ldo;
    return r;
  };
  group(1);
  rc = conv_problem(g.p[0], W.hA, d, W16(Lw.conv1_w), 2 * d, F32(Lw.conv1_b), W.h1, 2 * d, P->bn_conv1);
  if (rc) return rc;
  rc = marked(launch_gemm_group(g, P->bn_conv1, sms, st), 1);
  if (rc) return rc;
  group(2);
  rc |= conv_problem(g.p[0], W.h1, 2 * d, W16(Lw.conv2c_w), d, F32(Lw.conv2c_b), W.hc2, d, P->bn_conv2);
  rc |= conv_problem(g.p[1], W.h1 + d, 2 * d, W16(Lw.conv2s_w), d, F32(Lw.conv2s_b), W.hs2, d, P->bn_conv2);
  if (rc) return rc;
  rc = marked(launch_gemm_group(g, P->bn_conv2, sms, st), 1);
  if (rc) return rc;
  {
    HeadFinalArgs a;
    a.h_cls = W.hc2;
    a.h_span = W.hs2;
    a.w_cls = F32(Lw.conv3c_w);
    a.w_span = F32(Lw.conv3s_w);
    a.b_cls = F32(Lw.conv3c_b);
    a.b_span = F32(Lw.conv3s_b);
    a.pred_logits = pred_logits;
    a.pred_spans = pred_spans;
    a.B = P->B;
    a.Lv = Lv;
    a.d = d;
    a.fmt = fmt;
    a.split = split;
    a.lo = ws_lo;
    rc = marked(launch_conv_head_final(a, st), 0);
    if (rc) return rc;
  }
  {
    PoolSalArgs a;
    a.x_txt = W.txtproj32;
    a.x_vid = vid_mem_proj;
    a.txt_mask = src_txt_mask;
    a.vid_mask = src_vid_mask;
    a.w = F32(Lw.pool_w);
    a.pooled = txt_mem_proj;
    a.saliency = saliency_scores;
    a.alpha_out = W.pool_alpha;
    a.logits_ws = W.pool_logits;
    a.B = P->B;
    a.Lt = Lt;
    a.Lv = Lv;
    a.d = d;
    rc = marked(launch_pool_saliency(a, st), 0);
    if (rc) return rc;
  }
  if (W.pred_logits) {  // keep the small outputs the backward needs (the caller owns the returned tensors and may free them)
    cudaMemcpyAsync(W.pred_logits, pred_logits, (size_t)P->Mv * 4, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(W.pred_spans, pred_spans, (size_t)P->Mv * 8, cudaMemcpyDeviceToDevice, st);
  }
  return 0;
}

extern "C" {

int univtg_forward(univtg_plan* P, const float* src_txt, const float* src_txt_mask, const float* src_vid,
                   const float* src_vid_mask, const float* droppath_scale, float* pred_logits, float* pred_spans,
                   float* vid_mem_proj, float* txt_mem_proj, float* saliency_scores, void* stream) {
  if (!P || !src_txt || !src_txt_mask || !src_vid || !src_vid_mask || !pred_logits || !pred_spans || !vid_mem_proj ||
      !txt_mem_proj || !saliency_scores) {
    set_error("univtg_forward: null argument");
    return 1;
  }
  return run_forward(P, make_infer_ws(P->cfg, P->shp, P->lay, P->ws), src_txt, src_txt_mask, src_vid, src_vid_mask, droppath_scale,
                     nullptr, nullptr, pred_logits, pred_spans, vid_mem_proj, txt_mem_proj, saliency_scores, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// single operators
// ------------------------------------------------------------------------------------------------
static int op_gemm_impl(const void* a, const void* b, int32_t M, int32_t N, int32_t K, int32_t a_mn, int32_t b_mn, int32_t fmt,
                        int32_t bn, int32_t ksplit, const float* bias, int32_t act, float alpha, float* out32, void* out16,
                        int32_t cluster, void* stream) {
  if (!a || !b || M < 1 || N < 1 || K < 1 || bn < 32 || bn > 256 || bn % 16 != 0) {
    set_error("univtg_op_gemm: bad argument");
    return 1;
  }
  if (cluster == 2 && b_mn) {
    set_error("univtg_op_gemm_cluster: cluster launches need a K-major B operand (b_mn = 0)");
    return 1;
  }
  const bool split = fmt == 2;
  if (split && (a_mn || b_mn || cluster == 2)) {
    set_error("univtg_op_gemm: fmt 2 (fp16x3) needs K-major A and B (a_mn = b_mn = 0) and no cluster");
    return 1;
  }
  if (split && ksplit > 1 && out16) {
    set_error("univtg_op_gemm: fmt 2 (fp16x3) out16 cannot be combined with ksplit > 1");
    return 1;
  }
  GemmGroup g;
  reset_group(g, 1, split ? 0 : fmt, split ? 1 : 0, split ? (long long)M * N : 0);
  g.cluster = cluster;
  GemmProblem& p = g.p[0];
  const uint16_t *a16 = reinterpret_cast<const uint16_t*>(a), *b16 = reinterpret_cast<const uint16_t*>(b);
  const Mat16 A = a_mn ? Mat16{a16, K, M, M} : Mat16{a16, M, K, K};
  const Mat16 Bm = b_mn ? Mat16{b16, K, N, N} : Mat16{b16, N, K, K};
  const int rc = setup_gemm(p, A, a_mn, Bm, b_mn, M, N, K, cluster == 2 ? bn / 2 : bn, split ? (long long)M * K : 0,
                            split ? (long long)N * K : 0);
  if (rc) return rc;
  p.ksplit = ksplit < 1 ? 1 : ksplit;
  p.bias = bias;
  p.act = act;
  p.alpha = alpha;
  p.out32 = out32;
  p.ld32 = N;
  p.out16 = reinterpret_cast<uint16_t*>(out16);
  p.ld16 = N;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return launch_gemm_group(g, bn, sms, (cudaStream_t)stream);
}

int univtg_op_gemm(const void* a, const void* b, int32_t M, int32_t N, int32_t K, int32_t a_mn, int32_t b_mn, int32_t fmt,
                   int32_t bn, int32_t ksplit, const float* bias, int32_t act, float alpha, float* out32, void* out16,
                   void* stream) {
  return op_gemm_impl(a, b, M, N, K, a_mn, b_mn, fmt, bn, ksplit, bias, act, alpha, out32, out16, 1, stream);
}

int univtg_op_gemm_cluster(const void* a, const void* b, int32_t M, int32_t N, int32_t K, int32_t a_mn, int32_t b_mn,
                           int32_t fmt, int32_t bn, int32_t ksplit, const float* bias, int32_t act, float alpha, float* out32,
                           void* out16, void* stream) {
  return op_gemm_impl(a, b, M, N, K, a_mn, b_mn, fmt, bn, ksplit, bias, act, alpha, out32, out16, 2, stream);
}

int univtg_debug_choose_tile(const int32_t* Ms, const int32_t* Ns, const int32_t* kblocks, int32_t num, int32_t num_sms, int32_t step,
                              int32_t max_split, int32_t* bn, int32_t* ksplit) {
  if (!Ms || !Ns || !kblocks || !bn || !ksplit || num < 1 || num > GEMM_MAX_GROUP || num_sms < 1 || (step != 16 && step != 64) || max_split < 1) {
    set_error("univtg_debug_choose_tile: bad argument");
    return 1;
  }
  const int32_t limits[GEMM_MAX_GROUP] = {max_split, max_split, max_split, max_split};
  const uv::TileChoice t = uv::choose_tile(Ms, Ns, kblocks, limits, num, num_sms, step);
  *bn = t.bn;
  *ksplit = t.ksplit;
  return 0;
}

int univtg_debug_choose_tile_group(const int32_t* Ms, const int32_t* Ns, const int32_t* kblocks, const int32_t* max_split, int32_t num,
                                   int32_t num_sms, int32_t step, int32_t* bn, int32_t* ksplit) {
  bool ok = Ms && Ns && kblocks && max_split && bn && ksplit && num >= 1 && num <= GEMM_MAX_GROUP && num_sms >= 1 && (step == 16 || step == 64);
  for (int p = 0; ok && p < num; ++p) ok = max_split[p] >= 1 && (max_split[p] & (max_split[p] - 1)) == 0;
  if (!ok) {
    set_error("univtg_debug_choose_tile_group: bad argument");
    return 1;
  }
  const uv::TileChoice t = uv::choose_tile(Ms, Ns, kblocks, max_split, num, num_sms, step);
  *bn = t.bn;
  for (int p = 0; p < num; ++p) ksplit[p] = t.ks[p];
  return 0;
}

int32_t univtg_debug_gemm_deal(const int32_t* Ms, const int32_t* Ns, const int32_t* kblocks, const int32_t* ksplit, int32_t num,
                               int32_t num_sms, int32_t bn, int32_t* cta, int32_t cap) {
  const int n = (Ms && Ns && kblocks && ksplit && (cta || cap == 0) && cap >= 0) ? uv::gemm_deal_ctas(Ms, Ns, kblocks, ksplit, num, num_sms, bn, cta, cap) : -1;
  if (n < 0) set_error("univtg_debug_gemm_deal: bad argument");
  return n;
}

int univtg_debug_gemm_timeline(void* buf) {
  uv::set_gemm_timeline_buffer(reinterpret_cast<unsigned long long*>(buf));
  return 0;
}

int univtg_op_layernorm(const float* in, int32_t rows, int32_t d, const float* gamma, const float* beta, float eps,
                        int32_t fmt, float* out32, void* out16, int32_t ld16, void* stream) {
  if (!in || !gamma || !beta || rows < 1 || d < 1) {
    set_error("univtg_op_layernorm: bad argument");
    return 1;
  }
  LnArgs a;
  memset(&a, 0, sizeof(a));
  a.in = in;
  a.ld_in = d;
  a.rows = rows;
  a.d = d;
  a.gamma = gamma;
  a.beta = beta;
  a.eps = eps;
  a.fmt = fmt == 2 ? 0 : fmt;
  a.out32 = out32;
  a.out16 = reinterpret_cast<uint16_t*>(out16);
  a.ld16 = out16 ? ld16 : d;
  a.split = fmt == 2;
  a.lo = fmt == 2 ? (long long)rows * a.ld16 : 0;
  return launch_layernorm(a, (cudaStream_t)stream);
}

// ---- single forward operators: thin wrappers over the launchers run_forward uses; each checks on the host what its kernel assumes and
// its routing does not (the vector kernels load fp32 operands as float4 and 16-bit ones as uint2). ----
int univtg_op_layernorm_fwd(const univtg_ln_fwd* q, const univtg_rng* rng, int32_t mask_index, int32_t* kernel_used, void* stream) {
  const char* fn = "univtg_op_layernorm_fwd";
  UV_REQ(q != nullptr, "%s: null args", fn);
  UV_REQ((q->in || q->in16) && q->gamma && q->beta, "%s: null in / in16, gamma or beta", fn);
  UV_REQ(q->rows >= 1 && q->d >= 1, "%s: rows %d / d %d", fn, q->rows, q->d);
  UV_REQ(q->ld_in >= q->d, "%s: ld_in %d smaller than d %d", fn, q->ld_in, q->d);
  UV_REQ(!q->in16 || q->in_fmt == 0 || q->in_fmt == 1, "%s: in_fmt %d (0 fp16, 1 bf16)", fn, q->in_fmt);
  UV_REQ(q->fmt >= 0 && q->fmt <= 2, "%s: fmt %d (0 fp16, 1 bf16, 2 fp16x3)", fn, q->fmt);
  UV_REQ(!q->add16 || q->ld_add16 >= q->d, "%s: ld_add16 %d smaller than d %d", fn, q->ld_add16, q->d);
  UV_REQ(!q->add16 || q->d % 4 != 0 || q->ld_add16 % 4 == 0, "%s: ld_add16 %d must be a multiple of 4 (64-bit loads)", fn, q->ld_add16);
  UV_REQ(!q->sum_out || q->add16, "%s: sum_out needs add16", fn);
  UV_REQ(!(q->out16 || q->out16p) || q->ld16 >= q->d, "%s: ld16 %d smaller than d %d", fn, q->ld16, q->d);
  UV_REQ(q->L >= 0 && q->Lv >= 0 && q->Lv <= q->L && (q->L == 0 || q->rows % q->L == 0), "%s: L %d / Lv %d (rows %% L == 0)", fn, q->L,
         q->Lv);
  UV_REQ(!(q->pos || q->pos_txt || q->outc) || q->L >= 1, "%s: pos, pos_txt and outc need the token structure (L >= 1)", fn);
  UV_REQ(!q->pos || q->out16p, "%s: pos is only used with out16p", fn);
  UV_REQ(q->fmt != 2 || (q->lo > 0 && q->lo % 4 == 0), "%s: fmt 2 needs lo > 0, a multiple of 4", fn);
  UV_REQ(q->fmt != 2 || (!q->mul32 && !(rng && rng->input_dropout > 0.f)), "%s: fmt 2 (fp16x3) takes no dropout (mul32 / rng)", fn);
  UV_REQ(!rng || !(rng->input_dropout > 0.f) || mask_index >= 0, "%s: mask_index %d", fn, mask_index);
  UV_REQ(al_(q->in, 16) && al_(q->gamma, 16) && al_(q->beta, 16) && al_(q->sum_out, 16) && al_(q->out32, 16) && al_(q->pos, 16) &&
             al_(q->pos_txt, 16) && al_(q->mul32, 16) && al_(q->mean_out, 4) && al_(q->rstd_out, 4),
         "%s: fp32 pointers must be 16-byte aligned", fn);
  UV_REQ(al_(q->in16, 8) && al_(q->add16, 8) && al_(q->out16, 8) && al_(q->out16p, 8) && al_(q->outc, 8),
         "%s: in16, add16, out16, out16p and outc must be 8-byte aligned", fn);
  LnArgs a;
  memset(&a, 0, sizeof(a));
  a.in = q->in;
  a.ld_in = q->ld_in;
  a.in16 = reinterpret_cast<const uint16_t*>(q->in16);
  a.in_fmt = q->in_fmt;
  a.add16 = reinterpret_cast<const uint16_t*>(q->add16);
  a.ld_add16 = q->ld_add16;
  a.sum_out = q->sum_out;
  a.rows = q->rows;
  a.d = q->d;
  a.gamma = q->gamma;
  a.beta = q->beta;
  a.eps = q->eps;
  a.fmt = q->fmt == 2 ? 0 : q->fmt;
  a.split = q->fmt == 2;
  a.lo = q->fmt == 2 ? (long long)q->lo : 0;
  a.L = q->L;
  a.Lv = q->Lv;
  a.out32 = q->out32;
  a.out16 = reinterpret_cast<uint16_t*>(q->out16);
  a.out16p = reinterpret_cast<uint16_t*>(q->out16p);
  a.ld16 = (q->out16 || q->out16p) ? q->ld16 : q->d;
  a.pos = q->pos;
  a.pos_txt = q->pos_txt;
  a.outc = reinterpret_cast<uint16_t*>(q->outc);
  a.mul32 = q->mul32;
  if (!a.mul32 && rng && rng->input_dropout > 0.f) a.drop = make_drop_spec(rng->seed, (unsigned int)mask_index, rng->input_dropout);
  a.mean_out = q->mean_out;
  a.rstd_out = q->rstd_out;
  int used = -1;
  const int rc = launch_layernorm(a, (cudaStream_t)stream, &used);
  if (kernel_used) *kernel_used = used;
  return rc;
}

int univtg_op_txt_pos(const univtg_txt_pos_fwd* q, const univtg_rng* rng, int32_t mask_index, void* stream) {
  const char* fn = "univtg_op_txt_pos";
  UV_REQ(q != nullptr, "%s: null args", fn);
  UV_REQ(q->xt && q->table && q->gamma && q->beta && q->pos && q->xpos16, "%s: null xt, table, gamma, beta, pos or xpos16", fn);
  UV_REQ((q->mean_out == nullptr) == (q->rstd_out == nullptr), "%s: mean_out and rstd_out must both be given or both be NULL", fn);
  UV_REQ(q->B >= 1 && q->Lt >= 1 && q->Lv >= 0 && q->L >= q->Lv + q->Lt, "%s: B %d / Lt %d / L %d / Lv %d (L >= Lv + Lt)", fn, q->B,
         q->Lt, q->L, q->Lv);
  UV_REQ(q->fmt >= 0 && q->fmt <= 2, "%s: fmt %d (0 fp16, 1 bf16, 2 fp16x3)", fn, q->fmt);
  UV_REQ(q->fmt != 2 || (q->lo > 0 && q->lo % 2 == 0), "%s: fmt 2 needs lo > 0, a multiple of 2", fn);
  UV_REQ(q->fmt != 2 || (!q->mul32 && !(rng && rng->input_dropout > 0.f)), "%s: fmt 2 (fp16x3) takes no dropout (mul32 / rng)", fn);
  UV_REQ(!rng || !(rng->input_dropout > 0.f) || mask_index >= 0, "%s: mask_index %d", fn, mask_index);
  UV_REQ(al_(q->xt, 8) && al_(q->table, 8) && al_(q->gamma, 8) && al_(q->beta, 8) && al_(q->mul32, 8) && al_(q->pos, 8) &&
             al_(q->mean_out, 4) && al_(q->rstd_out, 4) && al_(q->xpos16, 4),
         "%s: fp32 pointers must be 8-byte and xpos16 4-byte aligned", fn);
  TxtPosArgs a;
  memset(&a, 0, sizeof(a));
  a.xt = q->xt;
  a.table = q->table;
  a.gamma = q->gamma;
  a.beta = q->beta;
  a.mul32 = q->mul32;
  if (!a.mul32 && rng && rng->input_dropout > 0.f) a.drop = make_drop_spec(rng->seed, (unsigned int)mask_index, rng->input_dropout);
  a.pos = q->pos;
  a.mean_out = q->mean_out;
  a.rstd_out = q->rstd_out;
  a.xpos16 = reinterpret_cast<uint16_t*>(q->xpos16);
  a.B = q->B;
  a.Lt = q->Lt;
  a.L = q->L;
  a.Lv = q->Lv;
  a.d = q->d;
  a.fmt = q->fmt == 2 ? 0 : q->fmt;
  a.split = q->fmt == 2;
  a.lo = q->fmt == 2 ? (long long)q->lo : 0;
  return launch_txt_pos(a, (cudaStream_t)stream);
}

int univtg_op_sine_pos(const float* vid_mask, const float* txt_mask, const float* dim_t, float* pos, float* key_mask, int32_t B, int32_t Lv,
                       int32_t Lt, int32_t d, const univtg_rng* rng, int32_t n_sites, float* dp_out, void* stream) {
  const char* fn = "univtg_op_sine_pos";
  UV_REQ(vid_mask && dim_t && pos, "%s: null vid_mask, dim_t or pos", fn);
  UV_REQ(B >= 1 && Lv >= 1 && Lv <= 12288 && Lt >= 0, "%s: B %d / Lv %d / Lt %d (1 <= Lv <= 12288)", fn, B, Lv, Lt);
  UV_REQ(d >= 2 && d % 2 == 0, "%s: d %d must be even (sin / cos column pairs)", fn, d);
  UV_REQ(!key_mask || Lt == 0 || txt_mask, "%s: key_mask needs txt_mask", fn);
  UV_REQ(!dp_out || (rng && n_sites >= 1), "%s: dp_out needs rng and n_sites >= 1", fn);
  UV_REQ(al_(pos, 8) && al_(vid_mask, 4) && al_(txt_mask, 4) && al_(dim_t, 4) && al_(key_mask, 4) && al_(dp_out, 4),
         "%s: pos must be 8-byte aligned", fn);
  return launch_sine_pos(vid_mask, txt_mask, dim_t, pos, key_mask, B, Lv, Lt, d, (cudaStream_t)stream, dp_out, dp_out ? n_sites : 0,
                         rng ? rng->seed : 0ull, rng ? 1.0f - rng->droppath : 1.f);
}

int univtg_op_pool_saliency(const float* x_txt, const float* x_vid, const float* txt_mask, const float* vid_mask, const float* w,
                            float* pooled, float* saliency, float* alpha_out, float* logits, int32_t B, int32_t Lt, int32_t Lv, int32_t d,
                            void* stream) {
  const char* fn = "univtg_op_pool_saliency";
  UV_REQ(x_txt && x_vid && txt_mask && vid_mask && w && pooled && saliency && logits, "%s: null pointer argument", fn);
  UV_REQ(B >= 1 && Lt >= 1 && Lt <= 12288 && Lv >= 1, "%s: B %d / Lt %d / Lv %d (1 <= Lt <= 12288)", fn, B, Lt, Lv);
  UV_REQ(d >= 4 && d % 4 == 0, "%s: d %d must be a positive multiple of 4 (128-bit loads)", fn, d);
  UV_REQ(al_(x_txt, 16) && al_(x_vid, 16) && al_(w, 16) && al_(pooled, 16) && al_(saliency, 4) && al_(alpha_out, 4) && al_(logits, 4) &&
             al_(txt_mask, 4) && al_(vid_mask, 4),
         "%s: x_txt, x_vid, w and pooled must be 16-byte aligned", fn);
  PoolSalArgs a;
  a.x_txt = x_txt;
  a.x_vid = x_vid;
  a.txt_mask = txt_mask;
  a.vid_mask = vid_mask;
  a.w = w;
  a.pooled = pooled;
  a.saliency = saliency;
  a.alpha_out = alpha_out;
  a.logits_ws = logits;
  a.B = B;
  a.Lt = Lt;
  a.Lv = Lv;
  a.d = d;
  return launch_pool_saliency(a, (cudaStream_t)stream);
}

int univtg_op_conv_head_final(const void* h_cls, const void* h_span, const float* w_cls, const float* w_span, const float* b_cls,
                              const float* b_span, float* pred_logits, float* pred_spans, int32_t B, int32_t Lv, int32_t d, int32_t fmt,
                              void* stream) {
  const char* fn = "univtg_op_conv_head_final";
  UV_REQ(h_cls && h_span && w_cls && w_span && b_cls && b_span && pred_logits && pred_spans, "%s: null pointer argument", fn);
  UV_REQ(B >= 1 && Lv >= 1, "%s: B %d / Lv %d", fn, B, Lv);
  UV_REQ(d >= 2 && d % 2 == 0, "%s: d %d must be even (32-bit loads)", fn, d);
  UV_REQ(fmt >= 0 && fmt <= 2, "%s: fmt %d (0 fp16, 1 bf16, 2 fp16x3)", fn, fmt);
  UV_REQ(al_(h_cls, 4) && al_(h_span, 4) && al_(w_cls, 4) && al_(w_span, 4) && al_(b_cls, 4) && al_(b_span, 4) && al_(pred_logits, 4) &&
             al_(pred_spans, 4),
         "%s: h_cls / h_span must be 4-byte aligned", fn);
  HeadFinalArgs a;
  a.h_cls = reinterpret_cast<const uint16_t*>(h_cls);
  a.h_span = reinterpret_cast<const uint16_t*>(h_span);
  a.w_cls = w_cls;
  a.w_span = w_span;
  a.b_cls = b_cls;
  a.b_span = b_span;
  a.pred_logits = pred_logits;
  a.pred_spans = pred_spans;
  a.B = B;
  a.Lv = Lv;
  a.d = d;
  a.fmt = fmt == 2 ? 0 : fmt;
  a.split = fmt == 2;
  a.lo = fmt == 2 ? ((long long)B * (Lv + 1) + 2) * d : 0;
  return launch_conv_head_final(a, (cudaStream_t)stream);
}

int univtg_op_attention_fwd(const univtg_attn_fwd* q, const univtg_rng* rng, float p, int32_t layer, int32_t* kernel_used, void* stream) {
  const char* fn = "univtg_op_attention_fwd";
  UV_REQ(q != nullptr, "%s: null args", fn);
  UV_REQ(q->qkv && q->key_mask && q->out, "%s: null qkv, key_mask or out", fn);
  UV_REQ(q->B >= 1 && q->L >= 1 && q->H >= 1 && q->dh >= 1, "%s: B %d / L %d / H %d / dh %d", fn, q->B, q->L, q->H, q->dh);
  UV_REQ(q->fmt >= 0 && q->fmt <= 2, "%s: fmt %d (0 fp16, 1 bf16, 2 fp16x3)", fn, q->fmt);
  UV_REQ(q->impl == 0 || q->impl == 1, "%s: impl %d (0 tensor cores, 1 SIMT)", fn, q->impl);
  UV_REQ(q->impl == 1 || q->dh == 64 || q->dh == 128, "%s: tensor-core attention needs dh 64 or 128, got %d", fn, q->dh);
  UV_REQ(q->impl == 0 || q->L <= 12288, "%s: SIMT attention stages L %d <= 12288 scores per warp", fn, q->L);
  UV_REQ(!q->causal || (q->impl == 0 && q->dh == 64 && q->fmt != 2 && !(p > 0.f)), "%s: causal needs impl 0, dh 64, fmt 0/1, p 0", fn);
  UV_REQ(p >= 0.f && p < 1.f && (!(p > 0.f) || (rng && q->fmt != 2 && layer >= 0)), "%s: p %g needs rng, fmt 0/1 and layer >= 0", fn,
         (double)p);
  UV_REQ(al_(q->qkv, 16) && al_(q->out, 4) && al_(q->key_mask, 4) && al_(q->lse, 4), "%s: qkv must be 16-byte and out 4-byte aligned",
         fn);
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  const int d = q->H * q->dh;
  a.key_mask = q->key_mask;
  a.out = reinterpret_cast<uint16_t*>(q->out);
  a.lse = q->lse;
  a.scale = 1.0f / sqrtf((float)q->dh);
  a.B = q->B;
  a.L = q->L;
  a.H = q->H;
  a.dh = q->dh;
  a.d = d;
  a.fmt = q->fmt == 2 ? 0 : q->fmt;
  a.split = q->fmt == 2;
  a.causal = q->causal;
  if (a.split) {
    a.lo_qkv = (long long)q->B * q->L * 3 * d;
    a.lo_out = (long long)q->B * q->L * d;
  }
  if (p > 0.f) a.drop = make_drop_spec(rng->seed, (unsigned int)layer, p);
  if (kernel_used) *kernel_used = -1;
  if (q->impl == 1) return launch_attention_simt(a, reinterpret_cast<const uint16_t*>(q->qkv), (cudaStream_t)stream, kernel_used);
  if (make_tmap_op(&a.tm_qkv, q->qkv, (uint64_t)q->B * q->L, (uint64_t)3 * d, (uint64_t)3 * d, 128, 64, a.lo_qkv)) return 1;
  return launch_attention(a, (cudaStream_t)stream, kernel_used);
}

int univtg_op_attention(const void* qkv, const float* key_mask, void* out, float* lse, int32_t B, int32_t L, int32_t H,
                        int32_t dh, int32_t fmt, int32_t impl, void* stream) {
  if (!qkv || !key_mask || !out) {
    set_error("univtg_op_attention: null argument");
    return 1;
  }
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  const int d = H * dh;
  a.key_mask = key_mask;
  a.out = reinterpret_cast<uint16_t*>(out);
  a.lse = lse;
  a.scale = 1.0f / sqrtf((float)dh);
  a.B = B;
  a.L = L;
  a.H = H;
  a.dh = dh;
  a.d = d;
  a.fmt = fmt == 2 ? 0 : fmt;
  a.split = fmt == 2;
  if (a.split) {
    a.lo_qkv = (long long)B * L * 3 * d;
    a.lo_out = (long long)B * L * d;
  }
  if (impl == 1) return launch_attention_simt(a, reinterpret_cast<const uint16_t*>(qkv), (cudaStream_t)stream);
  if (make_tmap_op(&a.tm_qkv, qkv, (uint64_t)B * L, (uint64_t)3 * d, (uint64_t)3 * d, 128, 64, a.lo_qkv)) return 1;
  return launch_attention(a, (cudaStream_t)stream);
}

}  // extern "C"
