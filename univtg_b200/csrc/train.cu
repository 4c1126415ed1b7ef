// Training path of the C-ABI: the training workspace, the forward that keeps what backward needs (run_forward, api.cu), the
// backward pass (SURVEY.md A.6, reference main/train_vlp_ddp.py:56-64: outputs = model(...); losses.backward()) and the
// criterion entry points.  GEMM descriptors (tensor maps) are built per call; shapes vary per training batch anyway (collate
// pads to the batch max).
#include <stdlib.h>

#include "plan.h"

namespace {

// The training workspace: what the forward writes (one buffer per layer, FwdBufs) and the backward's scratch.
struct TrainWs : FwdBufs {
  float *vid_mem_proj, *txt_mem_proj;  // reserved beside the forward's pred_logits / pred_spans copies; not read
  float *dx, *dy, *dqkv32, *delta, *dz, *dxt_pool, *dA_v, *dA_t, *wtap;
  uint16_t *dbr16, *dhpre16, *dO16, *dqkv16, *dhc2, *dhs2, *dh1, *dxv16, *dxt16;
};

TrainWs make_train_ws(const univtg_config& c, const univtg_shape& s, const PackedLayout& L, uint8_t* base) {
  TrainWs w;
  memset(&w, 0, sizeof(w));
  Cursor cur;
  const size_t d = c.hidden_dim, ff = c.dim_feedforward, H = c.nheads;
  const size_t B = s.batch, Lv = s.l_vid, Lt = s.l_txt, Lc = Lv + Lt;
  const size_t M = B * Lc, Mv = B * Lv, Mt = B * Lt, Mh = B * (Lv + 1);
  auto take16 = [&](size_t elems) { return reinterpret_cast<uint16_t*>(base + cur.take(elems * 2)); };
  auto take32 = [&](size_t elems) { return reinterpret_cast<float*>(base + cur.take(elems * 4)); };
  size_t max_din_v = 0, max_din_t = 0;
  for (int i = 0; i < c.n_input_proj; ++i) {
    w.a_vid[i] = take16(Mv * L.vid[i].kpad);
    w.a_txt[i] = take16(Mt * L.txt[i].kpad);
    w.pmean_v[i] = take32(Mv);
    w.prstd_v[i] = take32(Mv);
    w.pmean_t[i] = take32(Mt);
    w.prstd_t[i] = take32(Mt);
    w.p_vid32[i] = take32(Mv * d);
    w.p_txt32[i] = take32(Mt * d);
    if ((size_t)L.vid[i].kpad > max_din_v) max_din_v = L.vid[i].kpad;
    if ((size_t)L.txt[i].kpad > max_din_t) max_din_t = L.txt[i].kpad;
  }
  w.txtproj32 = take32(Mt * d);
  w.pool_alpha = take32(B * Lt);
  w.pool_logits = take32(B * Lt);
  w.pos = take32(Mv * d);
  w.key_mask = take32(B * Lc);
  w.dp_scale = take32((size_t)2 * c.enc_layers * B);
  for (int l = 0; l <= c.enc_layers; ++l) {
    w.xin16[l] = take16(M * d);
    w.xpos16[l] = take16(M * d);
  }
  for (int l = 0; l < c.enc_layers; ++l) {
    w.qkv16[l] = take16(M * 3 * d);
    w.attn16[l] = take16(M * d);
    w.x1_16[l] = take16(M * d);
    w.h16[l] = take16(M * ff);
    w.lse[l] = take32(B * H * Lc);
    w.y1[l] = take32(M * d);
    w.mean1[l] = take32(M);
    w.rstd1[l] = take32(M);
    w.dgelu16[l] = take16(M * ff);
    w.y2[l] = take32(M * d);
    w.mean2[l] = take32(M);
    w.rstd2[l] = take32(M);
  }
  w.x32 = take32(M * d);
  w.x1_32 = take32(M * d);
  w.hA = take16((Mh + 2) * d);
  w.h1 = take16((Mh + 2) * 2 * d);
  w.hc2 = take16((Mh + 2) * d);
  w.hs2 = take16((Mh + 2) * d);
  w.br16 = take16(M * d);
  w.pred_logits = take32(Mv);
  w.pred_spans = take32(Mv * 2);
  w.vid_mem_proj = take32(Mv * d);
  w.txt_mem_proj = take32(B * d);
  w.dx = take32(M * d);
  w.dy = take32(M * d);
  w.dqkv32 = take32(M * 3 * d);
  w.delta = take32(B * H * Lc);
  w.dz = take32((Mh + 2) * 4);
  w.dxt_pool = take32(Mt * d);
  w.dA_v = take32(Mv * max_din_v);
  w.dA_t = take32(Mt * max_din_t);
  {  // tap-major planes of one conv weight gradient; also the K-padded copy of a projector weight gradient whose width is not a multiple of 8
    size_t n = (size_t)3 * d * d;
    if ((size_t)d * max_din_v > n) n = (size_t)d * max_din_v;
    if ((size_t)d * max_din_t > n) n = (size_t)d * max_din_t;
    w.wtap = take32(n);
  }
  w.dbr16 = take16(M * d);
  w.dhpre16 = take16(M * ff);
  w.dO16 = take16(M * d);
  w.dqkv16 = take16(M * 3 * d);
  w.dhc2 = take16((Mh + 2) * d);
  w.dhs2 = take16((Mh + 2) * d);
  w.dh1 = take16((Mh + 2) * 2 * d);
  w.dxv16 = take16(Mv * d);
  w.dxt16 = take16(Mt * d);
  w.total = cur.off;
  return w;
}

// Gradient operands use the plan's 16-bit format (one wgmma takes A and B in ONE format).  With fp16 they would
// underflow, so the whole backward runs on gradients multiplied by a power-of-two loss scale S: the upstream output
// gradients are scaled on entry, every intermediate stays scaled, and each PARAMETER gradient is multiplied by 1/S where it
// is written (GEMM alpha, column-sum / LayerNorm / head kernels).  bf16 plans simply use S = 1.

}  // namespace

extern "C" {

// Buffers whose untouched rows must read as zeros (conv-head layout [B*(Lv+1)+2, C]: the separator rows that implement the
// Conv1d zero padding, model/univtg.py:375-377).  Every other byte of a workspace is written by a kernel before it is read,
// so a pooled workspace only needs this when it is handed to a different shape (or for the first time).
int univtg_prepare_workspace(const univtg_config* cfg, const univtg_shape* shape, void* workspace, int32_t training_ws, void* stream) {
  if (!check_cfg(cfg) || !check_shape(shape) || !workspace) {
    if (workspace == nullptr) set_error("univtg_prepare_workspace: null workspace");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const PackedLayout L = make_layout(*cfg);
  const size_t d = cfg->hidden_dim, Mh = (size_t)shape->batch * (shape->l_vid + 1);
  uint8_t* base = reinterpret_cast<uint8_t*>(workspace);
  cudaError_t e = cudaSuccess;
  auto zero = [&](void* p, size_t bytes) {
    if (e == cudaSuccess) e = cudaMemsetAsync(p, 0, bytes, st);
  };
  auto zero_heads = [&](const FwdBufs& w) {
    zero(w.hA, (Mh + 2) * d * 2);
    zero(w.h1, (Mh + 2) * 2 * d * 2);
    zero(w.hc2, (Mh + 2) * d * 2);
    zero(w.hs2, (Mh + 2) * d * 2);
  };
  if (training_ws) {
    if (refuse_split(*cfg, "univtg_prepare_workspace (training workspace)")) return 1;
    const TrainWs T = make_train_ws(*cfg, *shape, L, base);
    zero_heads(T);
    zero(T.dhc2, (Mh + 2) * d * 2);
    zero(T.dhs2, (Mh + 2) * d * 2);
    zero(T.dh1, (Mh + 2) * 2 * d * 2);
  } else {
    const FwdBufs w = make_infer_ws(*cfg, *shape, L, base);
    zero_heads(w);
    if (is_split(*cfg)) zero_heads(make_infer_ws(*cfg, *shape, L, base + w.total));  // the lo planes
  }
  if (e != cudaSuccess) {
    set_error("univtg_prepare_workspace: %s", cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

size_t univtg_train_workspace_bytes(const univtg_config* cfg, const univtg_shape* shape) {
  if (!check_cfg(cfg) || !check_shape(shape) || refuse_split(*cfg, "univtg_train_workspace_bytes")) return 0;
  const int dh = cfg->hidden_dim / cfg->nheads, L = shape->l_vid + shape->l_txt;
  if (dh != 64 && dh != 128) {  // the SIMT attention backward holds a whole row of L scores per warp in shared memory
    const int max_L = attention_bwd_simt_max_L();
    if (L > max_L) {
      set_error("univtg_train_workspace_bytes: L = l_vid + l_txt = %d exceeds %d, the longest sequence the SIMT attention backward "
                "(head size %d, not 64 or 128) can stage in shared memory",
                L, max_L, dh);
      return 0;
    }
  }
  return make_train_ws(*cfg, *shape, make_layout(*cfg), nullptr).total;
}

// Training forward.  `ws` = training workspace (univtg_train_workspace_bytes, zero-filled once by the caller).
// drop_masks: HOST array of 2*n_input_proj device pointers (video layers, then text layers): fp32 [rows, din_i] input-dropout
// multipliers (0 or 1/(1-p)) or NULL entries / NULL array when dropout is off.
int univtg_forward_train(univtg_plan* P, void* ws, const float* src_txt, const float* src_txt_mask, const float* src_vid,
                         const float* src_vid_mask, const float* droppath_scale, const float* const* drop_masks,
                         const univtg_rng* rng, float* pred_logits, float* pred_spans, float* vid_mem_proj, float* txt_mem_proj,
                         float* saliency_scores, void* stream) {
  if (!P || !ws || !src_txt || !src_txt_mask || !src_vid || !src_vid_mask || !pred_logits || !pred_spans || !vid_mem_proj ||
      !txt_mem_proj || !saliency_scores) {
    set_error("univtg_forward_train: null argument");
    return 1;
  }
  if (refuse_split(P->cfg, "univtg_forward_train")) return 1;
  if (P->attn_dropout > 0.f && !rng) {
    set_error("univtg_forward_train: attention dropout p = %g needs an rng (its masks are drawn in-kernel)", (double)P->attn_dropout);
    return 1;
  }
  const TrainWs T = make_train_ws(P->cfg, P->shp, P->lay, reinterpret_cast<uint8_t*>(ws));
  const int rc = run_forward(P, T, src_txt, src_txt_mask, src_vid, src_vid_mask, droppath_scale, drop_masks, rng, pred_logits,
                             pred_spans, vid_mem_proj, txt_mem_proj, saliency_scores, (cudaStream_t)stream);
  if (rc) return rc;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("univtg_forward_train: %s", cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

// Backward of univtg_forward_train.  g_*: upstream gradients of the four differentiable outputs (NULL = zero).
// grads: HOST array of device pointers, one fp32 gradient tensor per parameter in univtg_pack_weights order; the tensors must
// be zero-filled by the caller (several are accumulated atomically); they are written in the parameters' native layouts.
// drop_masks / droppath_scale: the same arrays that were passed to the forward.
int univtg_backward(univtg_plan* P, void* ws, const float* src_txt, const float* src_vid, const float* droppath_scale,
                    const float* const* drop_masks, const univtg_rng* rng, const float* g_logits, const float* g_spans,
                    const float* g_vid_mem_proj, const float* g_txt_mem_proj, float grad_scale, float* const* grads,
                    int32_t n_grads, void* stream) {
  if (!P || !ws || !grads || !src_txt || !src_vid || !(grad_scale > 0.f)) {
    set_error("univtg_backward: null argument");
    return 1;
  }
  if (refuse_split(P->cfg, "univtg_backward")) return 1;
  const univtg_config& c = P->cfg;
  const ParamIndex ix(c);
  const int n_params = ix.count() + (P->txt_pos_on ? 3 : 0);  // + txt_position_embed.* with learned text positions
  if (n_grads != n_params) {
    set_error("univtg_backward: expected %d gradient tensors (text positions %s), got %d", n_params, P->txt_pos_on ? "on" : "off",
              n_grads);
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const PackedLayout& Lw = P->lay;
  const uint8_t* pk = P->packed;
  auto F32 = [&](size_t off) { return reinterpret_cast<const float*>(pk + off); };
  auto W16 = [&](size_t off) { return reinterpret_cast<const uint16_t*>(pk + off); };
  const TrainWs T = make_train_ws(c, P->shp, Lw, reinterpret_cast<uint8_t*>(ws));
  if (droppath_scale == nullptr && rng != nullptr && rng->droppath > 0.f) droppath_scale = T.dp_scale;  // drawn by the forward
  const bool drop_rng = drop_masks == nullptr && rng != nullptr && rng->input_dropout > 0.f;
  if (P->attn_dropout > 0.f && !rng) {
    set_error("univtg_backward: attention dropout p = %g needs the forward's rng", (double)P->attn_dropout);
    return 1;
  }
  const int d = P->d, ff = P->ff, fmt = c.operand_format, M = P->M, Mv = P->Mv, Mt = P->Mt, Mh = P->Mh, L = P->L, Lv = P->Lv,
            Lt = P->Lt, B = P->B;
  // persistent GEMM grids assume every CTA is resident at once; when a gradient all-reduce runs beside the backward its CTAs
  // hold some SMs, and a full-width grid would wait for them (a second wave): launch on the SMs that are left
  const int sms = (P->num_sms_bwd > 0 && P->num_sms_bwd < P->num_sms) ? P->num_sms_bwd : P->num_sms;
  const float GS = grad_scale;           // loss scale carried by every intermediate gradient
  const float INV = 1.0f / grad_scale;   // applied wherever a parameter gradient is written

  int rc = 0;
  GemmGroup g;
  const int np = c.n_input_proj;
  const bool txt_pos = P->txt_pos_on != 0;
  const TxtPosWs TP = txt_pos ? make_txt_pos_ws(c, P->shp, P->txt_pos.scratch) : TxtPosWs{};
  const TxtRows txt_rows = txt_pos ? TxtRows{TP.dqk16, L, Lv, 2 * d} : TxtRows{nullptr, 0, 0, 0};

  cudaMemsetAsync(T.dx, 0, (size_t)M * d * 4, st);

  // ================================================ heads ================================================
  if (g_logits && g_spans) {
    HeadFinalBwdArgs a;
    memset(&a, 0, sizeof(a));
    a.g_logits = g_logits;
    a.g_spans = g_spans;
    a.pred_logits = T.pred_logits;
    a.pred_spans = T.pred_spans;
    a.h_cls = T.hc2;
    a.h_span = T.hs2;
    a.w_cls = F32(Lw.conv3c_w);
    a.w_span = F32(Lw.conv3s_w);
    a.dz = T.dz;
    a.dh_cls = T.dhc2;
    a.dh_span = T.dhs2;
    a.gw_cls = grads[ix.cls(4)];
    a.gb_cls = grads[ix.cls(5)];
    a.gw_span = grads[ix.span(4)];
    a.gb_span = grads[ix.span(5)];
    a.cs_cls = grads[ix.cls(3)];   // bias gradient of class_embed.layers.1 = column sums of d(hidden 2)
    a.cs_span = grads[ix.span(3)];
    a.B = B;
    a.Lv = Lv;
    a.d = d;
    a.fmt_act = fmt;
    a.fmt_grad = fmt;
    a.in_scale = GS;
    a.pgrad_scale = INV;
    rc = launch_head_final_bwd(a, st);
    if (rc) return rc;

    // conv layout helpers (conv_dgrad_problem / conv_wgrad_problem, plan.h): buffer row = logical row + 1
    auto conv_dgrad = [&](GemmProblem& p, const uint16_t* dY, int ldy, int Kc /*out channels*/, const uint16_t* Wp /*[Kc, 3*Cin]*/,
                          int Cin, int bnn) -> int { return conv_dgrad_problem(p, Mh, dY, ldy, Kc, Wp, Cin, bnn); };
    // wgrad of one tap, written as a tap-major plane of T.wtap (launch_tap_interleave then builds the [N, C, 3] layout with 256-bit
    // stores here instead of stride-3 scalars)
    const TileChoice t_cw = tile_for(sms, 64, MNK{d, d, Mh, 8}, MNK{d, d, Mh, 8}, MNK{d, d, Mh, 8});
    auto conv_wgrad = [&](GemmProblem& p, const uint16_t* dY, int ldy, int Nc, const uint16_t* X, int ldx, int Cin, int t) -> int {
      const int r = conv_wgrad_problem(p, Mh, dY, ldy, Nc, X, ldx, Cin, t, t_cw.bn);
      p.out32 = T.wtap + (size_t)t * Nc * Cin;
      p.ld32 = Cin;
      p.alpha = INV;
      p.ksplit = t_cw.ks[t];
      return r;
    };
    const int bn_c2d = tile_for(sms, 64, MNK{Mh, d, 3 * d}, MNK{Mh, d, 3 * d}).bn;
    const int bn_c1d = tile_for(sms, 64, MNK{Mh, d, 6 * d}).bn;
    // (splitting the k-blocks of the layer-1 dgrad - 76 tiles of 96 k-blocks - over idle SMs saves ~8 us but reduces into the stream
    // gradient with atomics, which makes every gradient upstream of the heads order-dependent in its last bits: not taken)
    // ---- conv layer 2 (two heads): dgrad -> dh1 [Mh+2, 2d] (class cols [0,d), span cols [d,2d)), ReLU mask of h1 ----
    reset_group(g, 2, fmt);
    rc |= conv_dgrad(g.p[0], T.dhc2, d, d, W16(Lw.conv2c_w), d, bn_c2d);
    rc |= conv_dgrad(g.p[1], T.dhs2, d, d, W16(Lw.conv2s_w), d, bn_c2d);
    if (rc) return rc;
    for (int s = 0; s < 2; ++s) {
      GemmProblem& p = g.p[s];
      p.rps_in = Lv + 1;
      p.rps_out = Lv + 1;
      p.row_off = 1;
      p.zero_sep = 1;
      p.mask16 = T.h1 + s * d;
      p.ld_mask = 2 * d;
      p.out16 = T.dh1 + s * d;
      p.ld16 = 2 * d;
      p.colsum = grads[s == 0 ? ix.cls(1) : ix.span(1)];  // bias gradient of conv layer 0 (saves a separate column-sum pass)
      p.colsum_scale = INV;
    }
    rc = gemm_launch(P, g, bn_c2d, sms, st);
    if (rc) return rc;
    // wgrad conv layer 2: 2 heads x 3 taps
    for (int s = 0; s < 2; ++s) {
      reset_group(g, 3, fmt);
      for (int t = 0; t < 3; ++t)
        rc |= conv_wgrad(g.p[t], s == 0 ? T.dhc2 : T.dhs2, d, d, T.h1 + s * d, 2 * d, d, t);
      if (rc) return rc;
      if (t_cw.ksplit > 1) cudaMemsetAsync(T.wtap, 0, (size_t)3 * d * d * 4, st);  // split-K accumulates into the planes
      rc = gemm_launch(P, g, t_cw.bn, sms, st);
      if (rc) return rc;
      rc = launch_tap_interleave(T.wtap, grads[s == 0 ? ix.cls(2) : ix.span(2)], d, d, st);
      if (rc) return rc;
    }
    // ---- conv layer 1 (fused N = 2d): dgrad -> stream gradient of the video rows ----
    reset_group(g, 1, fmt);
    rc = conv_dgrad(g.p[0], T.dh1, 2 * d, 2 * d, W16(Lw.conv1_w), d, bn_c1d);
    if (rc) return rc;
    g.p[0].rps_in = Lv + 1;
    g.p[0].rps_out = L;
    g.p[0].row_off = 0;
    g.p[0].skip_sep = 1;
    g.p[0].out32 = T.dx;
    g.p[0].ld32 = d;
    rc = gemm_launch(P, g, bn_c1d, sms, st);
    if (rc) return rc;
    // wgrad conv layer 1: class rows [0,d) and span rows [d,2d) of the fused weight
    for (int s = 0; s < 2; ++s) {
      reset_group(g, 3, fmt);
      for (int t = 0; t < 3; ++t) rc |= conv_wgrad(g.p[t], T.dh1 + s * d, 2 * d, d, T.hA, d, d, t);
      if (rc) return rc;
      if (t_cw.ksplit > 1) cudaMemsetAsync(T.wtap, 0, (size_t)3 * d * d * 4, st);
      rc = gemm_launch(P, g, t_cw.bn, sms, st);
      if (rc) return rc;
      rc = launch_tap_interleave(T.wtap, grads[s == 0 ? ix.cls(0) : ix.span(0)], d, d, st);
      if (rc) return rc;
    }
  }

  // stage events: gradients of a parameter group are final once the stream reaches this point (univtg_backward_stages)
  auto stage_done = [&](int k) {
    if (P->n_grad_events > 0 && k < P->n_grad_events) cudaEventRecord(P->grad_events[k], st);
  };
  // attention pooling of the text tokens: needs only the loss gradient of the pooled vector, so it runs before the first stage
  // event and its weight gradient travels with the heads' slice
  if (g_txt_mem_proj) {
    PoolBwdArgs a;
    a.x_txt = T.txtproj32;
    a.alpha = T.pool_alpha;
    a.w = F32(Lw.pool_w);
    a.g_pooled = g_txt_mem_proj;
    a.dx_txt = T.dxt_pool;
    a.gw = grads[ix.pool()];
    a.out_scale = GS;
    a.B = B;
    a.Lt = Lt;
    a.d = d;
    rc = launch_pool_bwd(a, st);
    if (rc) return rc;
  }
  stage_done(0);  // conv heads + weightedpool.weight

  // ================================================ encoder ================================================
  // LayerNorm backward of a residual block: dx (grad of the LayerNorm output) -> dy (grad of x + s * branch), branch operand s * dy
  // in dbr16; parameter gradients dgamma / dbeta, and dbias = column sums of s * dy (bias gradient of the branch's last linear)
  auto ln_bwd = [&](const float* y, const float* mean, const float* rstd, const float* gamma, const float* s, float* dgamma,
                    float* dbeta, float* dbias) -> int {
    LnBwdArgs a;
    memset(&a, 0, sizeof(a));
    a.dout = T.dx;
    a.ld_dout = d;
    a.y = y;
    a.ld_y = d;
    a.mean = mean;
    a.rstd = rstd;
    a.gamma = gamma;
    a.rows = M;
    a.d = d;
    a.row_scale = s;
    a.L = L;
    a.dy32 = T.dy;
    a.dbr16 = T.dbr16;
    a.ld16 = d;
    a.fmt16 = fmt;
    a.dgamma = dgamma;
    a.dbeta = dbeta;
    a.colsum = dbias;
    a.pgrad_scale = INV;
    return launch_layernorm_bwd(a, st);
  };
  // Each data gradient shares one launch with the weight gradients that read the same gradient operand.  A d-wide data gradient
  // is a single wave that leaves SMs idle, and a weight gradient is a few long output tiles: dealt together longest first, the
  // weight gradients' units fill the SMs the data gradient leaves, with fewer split-K reductions (choose_tile picks each weight
  // gradient's split), and the launch ramps and tails of separate launches go away (DESIGN §5.1).  Every operand of a launch is
  // complete when it starts; no buffer is written by one problem of a launch and read or written by another.
  const TileChoice t_f2 = tile_for(sms, 64, MNK{M, ff, d}, MNK{d, ff, M, 4});  // FFN2 dgrad + linear2.weight
  const TileChoice t_f1 = tile_for(sms, 64, MNK{M, d, ff}, MNK{ff, d, M, 4});  // FFN1 dgrad + linear1.weight
  const TileChoice t_o = tile_for(sms, 64, MNK{M, d, d}, MNK{d, d, M, 4});     // out-proj dgrad + out_proj.weight
  // QKV dgrad (+ text-position dgrad) + the q|k and v rows of in_proj_weight
  const TileChoice t_q = txt_pos ? tile_for(sms, 64, MNK{M, d, 3 * d}, MNK{Mt, d, 2 * d}, MNK{2 * d, d, M, 4}, MNK{d, d, M, 4})
                                 : tile_for(sms, 64, MNK{M, d, 3 * d}, MNK{2 * d, d, M, 4}, MNK{d, d, M, 4});
  for (int l = c.enc_layers - 1; l >= 0; --l) {
    const LayerPacked& lp = Lw.layer[l];
    const float* s1 = droppath_scale ? droppath_scale + (size_t)(2 * l) * B : nullptr;
    const float* s2 = droppath_scale ? droppath_scale + (size_t)(2 * l + 1) * B : nullptr;
    // ---- LN2 backward: dx (grad of the layer output) -> dy (grad of x1 + s2 * F), branch operand s2 * dy ----
    rc = ln_bwd(T.y2[l], T.mean2[l], T.rstd2[l], F32(lp.n2w), s2, grads[ix.layer(l, 10)], grads[ix.layer(l, 11)],
                grads[ix.layer(l, 7)]);  // linear2.bias
    if (rc) return rc;
    // ---- FFN2: dgrad -> d(hpre) = (dF W2) * gelu'(hpre) (saved 16-bit derivative);  wgrad dW2 = dF^T h ----
    // ---- FFN1: dgrad d(x1) = dhpre W1 + dy (residual);          wgrad dW1 = dhpre^T x1 ----
    auto ffn2_dgrad = [&](GemmProblem& p, int bnn) -> int {
      int r = setup_gemm(p, Mat16{T.dbr16, M, d, d}, 0, Mat16{W16(lp.w2), d, ff, ff}, 1, M, ff, d, bnn);
      p.mask16 = T.dgelu16[l];  // d(hpre) = (dF W2) * GELU'(hpre), the derivative saved by the forward as a 16-bit operand
      p.ld_mask = ff;
      p.mask_mul = 1;
      p.out16 = T.dhpre16;
      p.ld16 = ff;
      p.colsum = grads[ix.layer(l, 5)];  // linear1.bias
      p.colsum_scale = INV;
      return r;
    };
    auto ffn2_wgrad = [&](GemmProblem& p, int bnn, int ks) -> int {
      int r = setup_gemm(p, Mat16{T.dbr16, M, d, d}, 1, Mat16{T.h16[l], M, ff, ff}, 1, d, ff, M, bnn);
      p.out32 = grads[ix.layer(l, 6)];  // linear2.weight [d, ff]
      p.ld32 = ff;
      p.alpha = INV;
      p.ksplit = ks;
      return r;
    };
    auto ffn1_dgrad = [&](GemmProblem& p, int bnn) -> int {
      int r = setup_gemm(p, Mat16{T.dhpre16, M, ff, ff}, 0, Mat16{W16(lp.w1), ff, d, d}, 1, M, d, ff, bnn);
      p.resid = T.dy;
      p.ld_resid = d;
      p.out32 = T.dx;
      p.ld32 = d;
      return r;
    };
    auto ffn1_wgrad = [&](GemmProblem& p, int bnn, int ks) -> int {
      int r = setup_gemm(p, Mat16{T.dhpre16, M, ff, ff}, 1, Mat16{T.x1_16[l], M, d, d}, 1, ff, d, M, bnn);
      p.out32 = grads[ix.layer(l, 4)];  // linear1.weight [ff, d]
      p.ld32 = d;
      p.alpha = INV;
      p.ksplit = ks;
      return r;
    };
    {  // FFN2 launch: reads dbr16, W2, dgelu16, h16; writes dhpre16, linear1.bias (column sums), linear2.weight
      reset_group(g, 2, fmt);
      rc |= ffn2_dgrad(g.p[0], t_f2.bn);
      rc |= ffn2_wgrad(g.p[1], t_f2.bn, t_f2.ks[1]);
      if (rc) return rc;
      rc = gemm_launch(P, g, t_f2.bn, sms, st);
      if (rc) return rc;
      // FFN1 launch: reads dhpre16, W1, dy, x1_16; writes dx, linear1.weight
      reset_group(g, 2, fmt);
      rc |= ffn1_dgrad(g.p[0], t_f1.bn);
      rc |= ffn1_wgrad(g.p[1], t_f1.bn, t_f1.ks[1]);
      if (rc) return rc;
      rc = gemm_launch(P, g, t_f1.bn, sms, st);
      if (rc) return rc;
    }
    // ---- LN1 backward ----
    rc = ln_bwd(T.y1[l], T.mean1[l], T.rstd1[l], F32(lp.n1w), s1, grads[ix.layer(l, 8)], grads[ix.layer(l, 9)],
                grads[ix.layer(l, 3)]);  // out_proj.bias
    if (rc) return rc;
    // ---- out-proj: dgrad -> dO (16-bit); wgrad dWo = dA^T attn ----
    auto out_dgrad = [&](GemmProblem& p, int bnn) -> int {
      int r = setup_gemm(p, Mat16{T.dbr16, M, d, d}, 0, Mat16{W16(lp.w_out), d, d, d}, 1, M, d, d, bnn);
      p.out16 = T.dO16;
      p.ld16 = d;
      return r;
    };
    auto out_wgrad = [&](GemmProblem& p, int bnn, int ks) -> int {
      int r = setup_gemm(p, Mat16{T.dbr16, M, d, d}, 1, Mat16{T.attn16[l], M, d, d}, 1, d, d, M, bnn);
      p.out32 = grads[ix.layer(l, 2)];
      p.ld32 = d;
      p.alpha = INV;
      p.ksplit = ks;
      return r;
    };
    {  // reads dbr16, W_out, attn16; writes dO16, out_proj.weight
      reset_group(g, 2, fmt);
      rc |= out_dgrad(g.p[0], t_o.bn);
      rc |= out_wgrad(g.p[1], t_o.bn, t_o.ks[1]);
      if (rc) return rc;
      rc = gemm_launch(P, g, t_o.bn, sms, st);
      if (rc) return rc;
    }
    // ---- attention core backward -> dqkv32 -> dqkv16 (+ in_proj_bias gradient) ----
    rc = launch_attn_delta(T.dO16, fmt, T.attn16[l], fmt, T.delta, B, L, P->H, P->dh, st);
    if (rc) return rc;
    bool fused16 = false;
    {
      AttnBwdArgs a = attention_bwd_args(T.qkv16[l], T.dO16, T.key_mask, T.lse[l], T.delta, T.dqkv32, B, L, P->H, P->dh, fmt);
      if (P->attn_dropout > 0.f) a.drop = plan_drop_spec(P, rng, (unsigned int)l, P->attn_dropout);  // the forward's masks
      // one key tile on tensor cores: the kernel emits the 16-bit operands itself (the in_proj_bias column sums are a separate pass)
      int dq_mode = 2;
      rc = attention_bwd_route(a, P->dh == 64 || P->dh == 128, T.dqkv16, st, &dq_mode, nullptr, P);
      if (rc) return rc;
      fused16 = dq_mode == 0;
    }
    // (with text positions the same pass also copies the text rows of [dq | dk] into TP.dqk16)
    if (!fused16) rc = launch_cvt16_colsum(T.dqkv32, 3 * d, T.dqkv16, 3 * d, M, 3 * d, fmt, grads[ix.layer(l, 1)], INV, st, txt_rows);
    else rc = launch_colsum16(T.dqkv16, 3 * d, M, 3 * d, fmt, grads[ix.layer(l, 1)], INV, st, txt_rows);  // in_proj_bias gradient
    if (rc) return rc;
    // ---- in-projections: dgrad dx = dy + [dq|dk|dv] [Wq;Wk;Wv]; wgrad dWqk = [dq|dk]^T (x+pos), dWv = dv^T x ----
    auto qkv_dgrad = [&](GemmProblem& p, int bnn) -> int {
      int r = setup_gemm(p, Mat16{T.dqkv16, M, 3 * d, 3 * d}, 0, Mat16{W16(lp.w_in), 3 * d, d, d}, 1, M, d, 3 * d, bnn);
      p.resid = T.dy;
      p.ld_resid = d;
      p.out32 = T.dx;
      p.ld32 = d;
      return r;
    };
    auto qkv_wgrads = [&](GemmProblem& pqk, GemmProblem& pv, int bnn, int ks_qk, int ks_v) -> int {
      int r = setup_gemm(pqk, Mat16{T.dqkv16, M, 2 * d, 3 * d}, 1, Mat16{T.xpos16[l], M, d, d}, 1, 2 * d, d, M, bnn);
      r |= setup_gemm(pv, Mat16{T.dqkv16 + 2 * d, M, d, 3 * d}, 1, Mat16{T.xin16[l], M, d, d}, 1, d, d, M, bnn);
      pqk.out32 = grads[ix.layer(l, 0)];
      pqk.ld32 = d;
      pv.out32 = grads[ix.layer(l, 0)] + (size_t)2 * d * d;
      pv.ld32 = d;
      pqk.alpha = pv.alpha = INV;
      pqk.ksplit = ks_qk;
      pv.ksplit = ks_v;
      return r;
    };
    {  // reads dqkv16, W_in, dy, xpos16, xin16 (text positions: dqk16, and dpos in its own problem's epilogue); writes dx,
       // in_proj_weight (text positions: dpos)
      const int w = txt_pos ? 2 : 1;  // first weight-gradient problem (order of t_q's problems)
      reset_group(g, w + 2, fmt);
      rc = qkv_dgrad(g.p[0], t_q.bn);
      if (rc) return rc;
      if (txt_pos) {  // d(pos_t) += [dq | dk] [Wq; Wk] over the text rows (the first layer differentiated overwrites)
        GemmProblem& p = g.p[1];
        rc = setup_gemm(p, Mat16{TP.dqk16, Mt, 2 * d, 2 * d}, 0, Mat16{W16(lp.w_in), 2 * d, d, d}, 1, Mt, d, 2 * d, t_q.bn);
        if (rc) return rc;
        p.resid = l == c.enc_layers - 1 ? nullptr : TP.dpos;
        p.ld_resid = d;
        p.out32 = TP.dpos;
        p.ld32 = d;
      }
      rc = qkv_wgrads(g.p[w], g.p[w + 1], t_q.bn, t_q.ks[w], t_q.ks[w + 1]);
      if (rc) return rc;
      rc = gemm_launch(P, g, t_q.bn, sms, st);
      if (rc) return rc;
    }
    stage_done(1 + (c.enc_layers - 1 - l));  // encoder layer l
  }

  // ================================================ projectors ================================================
  if (txt_pos) {  // LayerNorm (+ dropout) backward of pos_t: its three parameter gradients, and du into the text rows of dx
    const int base = ix.count();
    TxtPosBwdArgs a;
    memset(&a, 0, sizeof(a));
    a.dpos = TP.dpos;
    a.xt = T.txtproj32;
    a.table = P->txt_pos.table;
    a.gamma = P->txt_pos.ln_weight;
    a.mean = TP.mean;
    a.rstd = TP.rstd;
    a.mul32 = P->txt_pos.drop_mul;
    if (!a.mul32 && rng != nullptr && rng->input_dropout > 0.f)
      a.drop = plan_drop_spec(P, rng, (unsigned int)(2 * np), rng->input_dropout);
    a.dx = T.dx;
    a.dtable = grads[base];
    a.dgamma = grads[base + 1];
    a.dbeta = grads[base + 2];
    a.pgrad_scale = INV;
    a.B = B;
    a.Lt = Lt;
    a.L = L;
    a.Lv = Lv;
    a.d = d;
    rc = launch_txt_pos_bwd(a, st);
    if (rc) return rc;
  }
  // gradient w.r.t. the projected tokens = stream gradient rows + direct (saliency-loss) gradients (dxt_pool: written up front)
  // column sums = bias gradient of the last projector layer AND the token-type embedding rows
  float* const g_type = grads[ix.type()];
  rc = launch_stream_gather(T.dx, L, 0, g_vid_mem_proj, GS, T.dxv16, g_type + d, INV, B, Lv, d, fmt, st);
  if (rc) return rc;
  rc = launch_stream_gather(T.dx, L, Lv, g_txt_mem_proj ? T.dxt_pool : nullptr, 1.0f, T.dxt16, g_type, INV, B, Lt, d, fmt, st);
  if (rc) return rc;
  cudaMemcpyAsync(grads[ix.vid(np - 1, 3)], g_type + d, (size_t)d * 4, cudaMemcpyDeviceToDevice, st);
  cudaMemcpyAsync(grads[ix.txt(np - 1, 3)], g_type, (size_t)d * 4, cudaMemcpyDeviceToDevice, st);
  for (int i = np - 1; i >= 0; --i) {
    const int kpv = Lw.vid[i].kpad, kpt = Lw.txt[i].kpad, dinv = Lw.vid[i].din, dint = Lw.txt[i].din;
    // a width like 2818 would force scalar epilogue stores: write rows padded to kpad with 256-bit stores, then a pitched copy
    const bool pad_v = (dinv % 8) != 0;
    const int nv = pad_v ? kpv : dinv;  // the operand a_vid[i] is zero beyond dinv
    // wgrad: dW_i = dOut^T a_i (video + text).  dgrad: dA_i = dOut W_i (fp32, [rows, kpad_i]: N is padded to the packed weight's
    // K so the epilogue stays on its 128-bit path even for the 2818-wide video features; the padded columns are zeros).  The
    // input-dropout mask is applied by the LayerNorm backward when it loads dA.  Layer 0's weight gradients end a gradient stage
    // (the event below), so its data gradients follow in a launch of their own; a later layer's four problems share one launch
    // (reads dxv16, dxt16, a_vid, a_txt and the packed weights; writes the weight gradients, T.wtap, dA_v and dA_t).
    const bool merged = i > 0;
    const TileChoice t_pw = merged ? tile_for(sms, 64, MNK{d, nv, Mv, 4}, MNK{d, dint, Mt, 4}, MNK{Mv, kpv, d}, MNK{Mt, kpt, d})
                                   : tile_for(sms, 64, MNK{d, nv, Mv, 16}, MNK{d, dint, Mt, 16});
    const int bn_pd = merged ? t_pw.bn : tile_for(sms, 64, MNK{Mv, kpv, d}, MNK{Mt, kpt, d}).bn;
    auto proj_dgrads = [&](GemmProblem* p) -> int {
      int r = setup_gemm(p[0], Mat16{T.dxv16, Mv, d, d}, 0, Mat16{W16(Lw.vid[i].w16), d, kpv, kpv}, 1, Mv, kpv, d, bn_pd);
      r |= setup_gemm(p[1], Mat16{T.dxt16, Mt, d, d}, 0, Mat16{W16(Lw.txt[i].w16), d, kpt, kpt}, 1, Mt, kpt, d, bn_pd);
      p[0].out32 = T.dA_v;
      p[0].ld32 = kpv;
      p[1].out32 = T.dA_t;
      p[1].ld32 = kpt;
      return r;
    };
    reset_group(g, merged ? 4 : 2, fmt);
    rc |= setup_gemm(g.p[0], Mat16{T.dxv16, Mv, d, d}, 1, Mat16{T.a_vid[i], Mv, kpv, kpv}, 1, d, nv, Mv, t_pw.bn);
    rc |= setup_gemm(g.p[1], Mat16{T.dxt16, Mt, d, d}, 1, Mat16{T.a_txt[i], Mt, kpt, kpt}, 1, d, dint, Mt, t_pw.bn);
    if (merged) rc |= proj_dgrads(g.p + 2);
    if (rc) return rc;
    g.p[0].out32 = pad_v ? T.wtap : grads[ix.vid(i, 2)];
    g.p[0].ld32 = nv;
    g.p[1].out32 = grads[ix.txt(i, 2)];
    g.p[1].ld32 = dint;
    g.p[0].alpha = g.p[1].alpha = INV;
    g.p[0].ksplit = t_pw.ks[0];
    g.p[1].ksplit = t_pw.ks[1];
    if (pad_v && t_pw.ks[0] > 1) cudaMemsetAsync(T.wtap, 0, (size_t)d * kpv * 4, st);  // split-K accumulates into the padded copy
    rc = gemm_launch(P, g, t_pw.bn, sms, st);
    if (rc) return rc;
    if (pad_v)
      cudaMemcpy2DAsync(grads[ix.vid(i, 2)], (size_t)dinv * 4, T.wtap, (size_t)kpv * 4, (size_t)dinv * 4, (size_t)d,
                        cudaMemcpyDeviceToDevice, st);
    // every projector weight, the later layers' LayerNorm terms and all biases are final here; what follows only produces the
    // first layer's LayerNorm terms - the 11.5 MB video weight gradient need not wait for it to start its exchange
    if (i == 0) stage_done(c.enc_layers + 1);
    if (!merged) {
      reset_group(g, 2, fmt);
      rc = proj_dgrads(g.p);
      if (rc) return rc;
      rc = gemm_launch(P, g, bn_pd, sms, st);
      if (rc) return rc;
    }
    // LayerNorm_i backward: parameter gradients; for i > 0 also the gradient of the previous layer's ReLU output
    for (int s = 0; s < 2; ++s) {
      LnBwdArgs a;
      memset(&a, 0, sizeof(a));
      const ProjPacked& pp = s == 0 ? Lw.vid[i] : Lw.txt[i];
      a.dout = s == 0 ? T.dA_v : T.dA_t;
      a.ld_dout = pp.kpad;
      a.dout_mul = drop_masks ? drop_masks[s * np + i] : nullptr;
      if (drop_rng) a.drop = plan_drop_spec(P, rng, (unsigned int)(s * np + i), rng->input_dropout);
      a.y = i == 0 ? (s == 0 ? src_vid : src_txt) : (s == 0 ? T.p_vid32[i - 1] : T.p_txt32[i - 1]);
      if (i == 0 && P->in_fmt != 0) {
        a.y16 = reinterpret_cast<const uint16_t*>(a.y);
        a.y_fmt = P->in_fmt - 1;
      }
      a.ld_y = pp.din;
      a.mean = s == 0 ? T.pmean_v[i] : T.pmean_t[i];
      a.rstd = s == 0 ? T.prstd_v[i] : T.prstd_t[i];
      a.gamma = F32(pp.ln_w);
      a.rows = s == 0 ? Mv : Mt;
      a.d = pp.din;
      a.dgamma = grads[s == 0 ? ix.vid(i, 0) : ix.txt(i, 0)];
      a.dbeta = grads[s == 0 ? ix.vid(i, 1) : ix.txt(i, 1)];
      a.pgrad_scale = INV;
      if (i > 0) {
        a.relu_mask_y = 1;
        a.dbr16 = s == 0 ? T.dxv16 : T.dxt16;
        a.ld16 = d;
        a.fmt16 = fmt;
        a.colsum = grads[s == 0 ? ix.vid(i - 1, 3) : ix.txt(i - 1, 3)];
      }
      rc = launch_layernorm_bwd(a, st);
      if (rc) return rc;
    }
  }
  stage_done(c.enc_layers + 2);  // LayerNorm terms of the first projector layers
  prof_mark(P, st, 3);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("univtg_backward: %s", cudaGetErrorString(e));
    return (int)e;
  }
  return 0;
}

int univtg_backward_stages(const univtg_config* cfg, int32_t* ranges, int32_t max_stages) {
  if (univtg_num_params(cfg) < 0) return -1;
  const ParamIndex ix(*cfg);
  const int nl = cfg->enc_layers;
  const int n = nl + 3;
  if (ranges == nullptr) return n;
  if (max_stages < n) {
    set_error("univtg_backward_stages: need room for %d stages", n);
    return -1;
  }
  auto put = [&](int k, int a0, int a1, int b0, int b1) {
    ranges[4 * k + 0] = a0;
    ranges[4 * k + 1] = a1;
    ranges[4 * k + 2] = b0;
    ranges[4 * k + 3] = b1;
  };
  put(0, ix.span(0), ix.count(), 0, 0);  // span_embed + class_embed, weightedpool.weight
  for (int k = 0; k < nl; ++k) {
    const int l = nl - 1 - k;
    put(1 + k, ix.layer(l, 0), ix.layer(l + 1, 0), 0, 0);
  }
  put(nl + 1, ix.vid(0, 2), ix.txt(0, 0), ix.txt(0, 2), ix.type() + 1);  // everything but the first layers' LayerNorm terms
  put(nl + 2, ix.vid(0, 0), ix.vid(0, 2), ix.txt(0, 0), ix.txt(0, 2));   // those (final only after the last LayerNorm backward)
  return n;
}

int univtg_plan_set_backward_sm_budget(univtg_plan* plan, int32_t num_sms) {
  if (!plan || num_sms < 0) {
    set_error("univtg_plan_set_backward_sm_budget: bad argument");
    return 1;
  }
  plan->num_sms_bwd = num_sms;
  return 0;
}

int univtg_plan_set_grad_events(univtg_plan* plan, void* const* events, int32_t n) {
  if (!plan || n < 0 || n > 24 || (n > 0 && !events)) {
    set_error("univtg_plan_set_grad_events: bad argument");
    return 1;
  }
  if (n > 0 && n != plan->cfg.enc_layers + 3) {
    set_error("univtg_plan_set_grad_events: expected %d events (univtg_backward_stages), got %d", plan->cfg.enc_layers + 3, n);
    return 1;
  }
  plan->n_grad_events = n;
  for (int i = 0; i < n; ++i) plan->grad_events[i] = reinterpret_cast<cudaEvent_t>(events[i]);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// criterion (reference SetCriterion.forward, model/univtg.py:338-351, losses 'spans' + 'labels' + 'saliency')
// scratch: device buffer of univtg_loss_scratch_bytes(B, Lv); holds the per-loss gradients between forward and backward.
// ------------------------------------------------------------------------------------------------
namespace {
struct LossScratch {
  float *g_spans_b, *g_spans_g, *g_logits_f, *cos_in, *vnorm, *tnorm, *sim, *g_cos_in, *g_sim;
  size_t total;
};
LossScratch make_loss_scratch(int B, int Lv, uint8_t* base) {
  LossScratch s;
  Cursor cur;
  auto take32 = [&](size_t n) { return reinterpret_cast<float*>(base + cur.take(n * 4)); };
  const size_t n = (size_t)B * Lv;
  s.g_spans_b = take32(2 * n);
  s.g_spans_g = take32(2 * n);
  s.g_logits_f = take32(n);
  s.cos_in = take32(n);
  s.vnorm = take32(n);
  s.tnorm = take32(B);
  s.sim = take32((size_t)B * B);
  s.g_cos_in = take32(n);
  s.g_sim = take32((size_t)B * B);
  s.total = cur.off;
  return s;
}
}  // namespace

int univtg_op_attention_bwd(const void* qkv, const void* dO, const void* O, const float* key_mask, const float* lse,
                            float* delta_ws, float* dqkv32, int32_t B, int32_t L, int32_t H, int32_t dh, int32_t fmt_act,
                            int32_t impl, void* stream) {
  if (!qkv || !dO || !O || !key_mask || !lse || !delta_ws || !dqkv32) {
    set_error("univtg_op_attention_bwd: null argument");
    return 1;
  }
  if (refuse_fmt2(fmt_act, "univtg_op_attention_bwd")) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = launch_attn_delta(reinterpret_cast<const uint16_t*>(dO), fmt_act, reinterpret_cast<const uint16_t*>(O), fmt_act,
                             delta_ws, B, L, H, dh, st);
  if (rc) return rc;
  AttnBwdArgs a = attention_bwd_args(qkv, dO, key_mask, lse, delta_ws, dqkv32, B, L, H, dh, fmt_act);
  return attention_bwd_route(a, impl == 0, nullptr, st, nullptr);
}

int univtg_op_attn_delta(const void* dO, int32_t fmt_do, const void* O, int32_t fmt_o, float* delta, int32_t B, int32_t L, int32_t H,
                         int32_t dh, int32_t* vec_used, void* stream) {
  const char* fn = "univtg_op_attn_delta";
  UV_REQ(dO && O && delta, "%s: null dO, O or delta", fn);
  UV_REQ((fmt_do == 0 || fmt_do == 1) && (fmt_o == 0 || fmt_o == 1), "%s: fmt_do %d / fmt_o %d (0 fp16, 1 bf16)", fn, fmt_do, fmt_o);
  UV_REQ(B >= 1 && L >= 1 && H >= 1 && dh >= 1, "%s: B %d / L %d / H %d / dh %d must be positive", fn, B, L, H, dh);
  int vec = -1;
  const int rc = launch_attn_delta(reinterpret_cast<const uint16_t*>(dO), fmt_do, reinterpret_cast<const uint16_t*>(O), fmt_o, delta, B,
                                   L, H, dh, (cudaStream_t)stream, &vec);
  if (vec_used) *vec_used = vec;
  return rc;
}

int univtg_op_attention_bwd_full(const univtg_attn_bwd* q, const univtg_rng* rng, float p, int32_t layer, int32_t* kernel_used,
                                 int32_t* dq_mode, void* stream) {
  const char* fn = "univtg_op_attention_bwd_full";
  UV_REQ(q != nullptr, "%s: null args", fn);
  UV_REQ(q->qkv && q->dO && q->key_mask && q->lse && q->delta && q->dqkv32, "%s: null qkv, dO, key_mask, lse, delta or dqkv32", fn);
  UV_REQ(q->B >= 1 && q->L >= 1 && q->H >= 1 && q->dh >= 1, "%s: B %d / L %d / H %d / dh %d must be positive", fn, q->B, q->L, q->H,
         q->dh);
  UV_REQ(q->fmt == 0 || q->fmt == 1, "%s: fmt %d (0 fp16, 1 bf16)", fn, q->fmt);
  UV_REQ(q->impl == 0 || q->impl == 1, "%s: impl %d (0 tensor cores, 1 SIMT)", fn, q->impl);
  UV_REQ(q->impl == 1 || q->dh == 64 || q->dh == 128, "%s: tensor-core attention backward needs dh 64 or 128, got %d", fn, q->dh);
  UV_REQ(!q->dqkv16 || (q->impl == 0 && q->L <= 128), "%s: dqkv16 needs impl 0 and a single key tile (L %d <= 128)", fn, q->L);
  UV_REQ(al_(q->qkv, 16) && al_(q->dO, 16), "%s: qkv and dO must be 16-byte aligned", fn);
  UV_REQ(al_(q->key_mask, 4) && al_(q->lse, 4) && al_(q->delta, 4) && al_(q->dqkv32, 8) && al_(q->dqkv16, 4),
         "%s: key_mask / lse / delta must be 4-byte, dqkv32 8-byte and dqkv16 4-byte aligned", fn);
  UV_REQ(p >= 0.f && p < 1.f && (!(p > 0.f) || (rng && layer >= 0)), "%s: p %g must be in [0, 1) and p > 0 needs rng and layer >= 0",
         fn, (double)p);
  if (q->impl == 1) {
    const int max_L = attention_bwd_simt_max_L();
    UV_REQ(q->L <= max_L, "%s: SIMT backward stages 32 L bytes of shared memory: L %d exceeds %d", fn, q->L, max_L);
  }
  AttnBwdArgs a = attention_bwd_args(q->qkv, q->dO, q->key_mask, q->lse, q->delta, q->dqkv32, q->B, q->L, q->H, q->dh, q->fmt);
  if (p > 0.f) a.drop = make_drop_spec(rng->seed, (unsigned int)layer, p);
  if (kernel_used) *kernel_used = -1;
  return attention_bwd_route(a, q->impl == 0, reinterpret_cast<uint16_t*>(q->dqkv16), (cudaStream_t)stream, dq_mode, kernel_used);
}

// ---- single backward operators: thin wrappers over the launchers univtg_backward uses.  Each checks on the host what its kernel
// assumes (null pointers, vector widths, alignment, size limits; UV_REQ, plan.h) and names the offending argument before anything is
// launched. ----

int univtg_op_gemm_group(univtg_gemm_problem* problems, int32_t num, int32_t fmt, int32_t bn, int32_t cluster, int32_t* full,
                         void* stream) {
  const char* fn = "univtg_op_gemm_group";
  UV_REQ(problems != nullptr && num >= 1 && num <= GEMM_MAX_GROUP, "%s: problems must hold 1..%d entries", fn, GEMM_MAX_GROUP);
  if (refuse_fmt2(fmt, fn)) return 1;
  UV_REQ(fmt == 0 || fmt == 1, "%s: fmt %d (0 fp16, 1 bf16)", fn, fmt);
  UV_REQ(bn >= 32 && bn <= 256 && bn % 16 == 0, "%s: bn %d (multiple of 16 in [32, 256])", fn, bn);
  UV_REQ(cluster == 1 || cluster == 2, "%s: cluster %d (1 or 2)", fn, cluster);
  GemmGroup g;
  reset_group(g, num, fmt);
  g.cluster = cluster;
  for (int i = 0; i < num; ++i) {
    const univtg_gemm_problem& q = problems[i];
    GemmProblem& p = g.p[i];
    UV_REQ(q.a && q.b, "%s: problem %d: null a or b", fn, i);
    UV_REQ(q.M >= 1 && q.N >= 1 && q.K >= 1, "%s: problem %d: M, N, K must be >= 1", fn, i);
    UV_REQ(q.lda % 8 == 0 && q.ldb % 8 == 0 && al_(q.a, 16) && al_(q.b, 16), "%s: problem %d: lda / ldb must be multiples of 8 and a / b 16-byte aligned", fn, i);
    UV_REQ(q.ksplit >= 1, "%s: problem %d: ksplit %d", fn, i, q.ksplit);
    for (int f : {q.a_fmt, q.b_fmt, q.out_fmt}) UV_REQ(f >= -1 && f <= 1, "%s: problem %d: 16-bit format %d (-1, 0, 1)", fn, i, f);
    UV_REQ(q.act >= ACT_NONE && q.act <= ACT_GELU, "%s: problem %d: act %d", fn, i, q.act);
    UV_REQ(!q.dact16 || q.act == ACT_GELU, "%s: problem %d: dact16 needs act = 2 (GELU)", fn, i);
    UV_REQ(!q.mask_mul || q.mask16, "%s: problem %d: mask_mul needs mask16", fn, i);
    UV_REQ(!(q.zero_sep || q.skip_sep) || q.rps_in > 0, "%s: problem %d: zero_sep / skip_sep need rps_in > 0", fn, i);
    UV_REQ(q.rps_in >= 0 && (q.rps_in == 0 || q.rps_out >= q.rps_in) && q.row_off >= 0, "%s: problem %d: rps_in %d / rps_out %d / row_off %d",
           fn, i, q.rps_in, q.rps_out, q.row_off);
    UV_REQ(!q.addtab || q.out16p, "%s: problem %d: addtab is only used with out16p", fn, i);
    UV_REQ(!q.out32 || q.ld32 >= q.N, "%s: problem %d: ld32 %d < N %d", fn, i, q.ld32, q.N);
    UV_REQ(!q.out32_id || q.ld32_id >= q.N, "%s: problem %d: ld32_id %d < N %d", fn, i, q.ld32_id, q.N);
    UV_REQ(!(q.out16 || q.out16p) || q.ld16 >= q.N, "%s: problem %d: ld16 %d < N %d", fn, i, q.ld16, q.N);
    UV_REQ(!q.resid || q.ld_resid >= q.N, "%s: problem %d: ld_resid %d < N %d", fn, i, q.ld_resid, q.N);
    UV_REQ(!q.addtab || q.ld_addtab >= q.N, "%s: problem %d: ld_addtab %d < N %d", fn, i, q.ld_addtab, q.N);
    UV_REQ(!q.mask16 || q.ld_mask >= q.N, "%s: problem %d: ld_mask %d < N %d", fn, i, q.ld_mask, q.N);
    UV_REQ(!q.dact16 || q.ld_dact >= q.N, "%s: problem %d: ld_dact %d < N %d", fn, i, q.ld_dact, q.N);
    // scalar-path stores are element-wise; the vector paths are chosen by launch_gemm_group only where alignment allows them
    UV_REQ(al_(q.out32, 4) && al_(q.out32_id, 4) && al_(q.resid, 4) && al_(q.addtab, 4) && al_(q.colsum, 4) && al_(q.out16, 2) &&
               al_(q.out16p, 2) && al_(q.mask16, 2) && al_(q.dact16, 2),
           "%s: problem %d: misaligned epilogue pointer", fn, i);
    int rc = 0;
    if (q.conv == 1) {
      UV_REQ(!q.a_mn && q.b_mn && q.K % 64 == 0, "%s: problem %d: conv dgrad needs a_mn = 0, b_mn = 1 and K %% 64 == 0", fn, i);
      UV_REQ(q.ldb == 3 * q.N, "%s: problem %d: conv dgrad weight pitch ldb must be 3 N", fn, i);
      rc = conv_dgrad_problem(p, q.M, reinterpret_cast<const uint16_t*>(q.a), q.lda, q.K, reinterpret_cast<const uint16_t*>(q.b), q.N, bn);
    } else if (q.conv == 2) {
      UV_REQ(q.a_mn && q.b_mn && q.tap >= 0 && q.tap <= 2, "%s: problem %d: conv wgrad needs a_mn = b_mn = 1 and tap in 0..2", fn, i);
      rc = conv_wgrad_problem(p, q.K, reinterpret_cast<const uint16_t*>(q.a), q.lda, q.M, reinterpret_cast<const uint16_t*>(q.b), q.ldb,
                              q.N, q.tap, bn);
    } else if (q.conv == 3) {
      UV_REQ(!q.a_mn && !q.b_mn && q.K % 192 == 0, "%s: problem %d: forward conv needs a_mn = b_mn = 0 and K = 3 Cin with Cin %% 64 == 0",
             fn, i);
      UV_REQ(q.lda >= q.K / 3 && q.ldb == q.K, "%s: problem %d: forward conv needs lda >= Cin and weight pitch ldb = K", fn, i);
      UV_REQ(cluster == 1, "%s: problem %d: forward conv runs without clusters", fn, i);
      rc = conv_fwd_problem(p, q.M, reinterpret_cast<const uint16_t*>(q.a), q.lda, q.K / 3, reinterpret_cast<const uint16_t*>(q.b), q.N, bn);
    } else {
      UV_REQ(q.conv == 0, "%s: problem %d: conv %d (0 plain, 1 dgrad, 2 wgrad, 3 forward)", fn, i, q.conv);
      const Mat16 A = q.a_mn ? Mat16{reinterpret_cast<const uint16_t*>(q.a), q.K, q.M, q.lda}
                             : Mat16{reinterpret_cast<const uint16_t*>(q.a), q.M, q.K, q.lda};
      const Mat16 Bm = q.b_mn ? Mat16{reinterpret_cast<const uint16_t*>(q.b), q.K, q.N, q.ldb}
                              : Mat16{reinterpret_cast<const uint16_t*>(q.b), q.N, q.K, q.ldb};
      UV_REQ(A.ld >= A.cols && Bm.ld >= Bm.cols, "%s: problem %d: lda / ldb smaller than the operand's row length", fn, i);
      rc = setup_gemm(p, A, q.a_mn, Bm, q.b_mn, q.M, q.N, q.K, cluster == 2 && !q.b_mn ? bn / 2 : bn);
    }
    if (rc) return rc;
    p.a_fmt = q.a_fmt;
    p.b_fmt = q.b_fmt;
    p.ksplit = q.ksplit;
    p.out_fmt = q.out_fmt;
    p.bias = q.bias;
    p.act = q.act;
    p.alpha = q.alpha;
    p.row_scale = q.row_scale;
    p.rps_in = q.rps_in;
    p.rps_out = q.rps_out;
    p.row_off = q.row_off;
    p.zero_sep = q.zero_sep;
    p.skip_sep = q.skip_sep;
    p.resid = q.resid;
    p.ld_resid = q.ld_resid;
    p.addtab = q.addtab;
    p.ld_addtab = q.ld_addtab;
    p.out32 = q.out32;
    p.ld32 = q.ld32;
    p.out32_id = q.out32_id;
    p.ld32_id = q.ld32_id;
    p.out16 = reinterpret_cast<uint16_t*>(q.out16);
    p.out16p = reinterpret_cast<uint16_t*>(q.out16p);
    p.ld16 = q.ld16;
    p.accumulate = q.accumulate;
    p.mask16 = reinterpret_cast<const uint16_t*>(q.mask16);
    p.ld_mask = q.ld_mask;
    p.mask_mul = q.mask_mul;
    p.dact16 = reinterpret_cast<uint16_t*>(q.dact16);
    p.ld_dact = q.ld_dact;
    p.colsum = q.colsum;
    p.colsum_scale = q.colsum_scale;
  }
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int used_full = 0;
  const int rc = launch_gemm_group(g, bn, sms, (cudaStream_t)stream, &used_full);
  for (int i = 0; i < num; ++i) problems[i].vec_ok = g.p[i].vec_ok;
  if (full) *full = used_full;
  return rc;
}

int univtg_op_layernorm_bwd(const univtg_ln_bwd* q, const univtg_rng* rng, int32_t mask_index, int32_t* kernel_used, void* stream) {
  const char* fn = "univtg_op_layernorm_bwd";
  UV_REQ(q != nullptr, "%s: null args", fn);
  UV_REQ(q->dout && (q->y || q->y16) && q->mean && q->rstd && q->gamma, "%s: null dout, y / y16, mean, rstd or gamma", fn);
  UV_REQ(q->rows >= 1 && q->d >= 1 && q->d <= 3072, "%s: rows %d / d %d (d <= 3072)", fn, q->rows, q->d);
  UV_REQ(q->ld_dout >= q->d && q->ld_y >= q->d, "%s: ld_dout %d / ld_y %d smaller than d %d", fn, q->ld_dout, q->ld_y, q->d);
  UV_REQ(!q->dbr16 || q->ld16 >= q->d, "%s: ld16 %d smaller than d %d", fn, q->ld16, q->d);
  UV_REQ(!q->y16 || (!q->dy32 && !q->dbr16), "%s: a 16-bit y (y16) is only supported for parameter gradients (dy32 = dbr16 = NULL)", fn);
  UV_REQ(!q->row_scale || q->L >= 1, "%s: row_scale needs L >= 1", fn);
  if (refuse_fmt2(q->fmt16, fn) || refuse_fmt2(q->y_fmt, fn)) return 1;
  UV_REQ(q->fmt16 == 0 || q->fmt16 == 1, "%s: fmt16 %d", fn, q->fmt16);
  UV_REQ(q->y_fmt == 0 || q->y_fmt == 1, "%s: y_fmt %d", fn, q->y_fmt);
  UV_REQ(al_(q->dout, 4) && al_(q->y, 4) && al_(q->y16, 2) && al_(q->dbr16, 2) && al_(q->dy32, 4) && al_(q->dgamma, 4) &&
             al_(q->dbeta, 4) && al_(q->colsum, 4) && al_(q->dout_mul, 4),
         "%s: misaligned pointer", fn);
  UV_REQ(!rng || !(rng->input_dropout > 0.f) || mask_index >= 0, "%s: mask_index %d", fn, mask_index);
  LnBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.dout = q->dout;
  a.ld_dout = q->ld_dout;
  a.y = q->y16 ? reinterpret_cast<const float*>(q->y16) : q->y;
  a.ld_y = q->ld_y;
  a.y16 = reinterpret_cast<const uint16_t*>(q->y16);
  a.y_fmt = q->y_fmt;
  a.mean = q->mean;
  a.rstd = q->rstd;
  a.gamma = q->gamma;
  a.rows = q->rows;
  a.d = q->d;
  a.row_scale = q->row_scale;
  a.L = q->L;
  a.relu_mask_y = q->relu_mask_y;
  a.dy32 = q->dy32;
  a.dbr16 = reinterpret_cast<uint16_t*>(q->dbr16);
  a.ld16 = q->ld16;
  a.fmt16 = q->fmt16;
  a.dgamma = q->dgamma;
  a.dbeta = q->dbeta;
  a.colsum = q->colsum;
  a.pgrad_scale = q->pgrad_scale;
  a.dout_mul = q->dout_mul;
  if (!a.dout_mul && rng && rng->input_dropout > 0.f) a.drop = make_drop_spec(rng->seed, (unsigned int)mask_index, rng->input_dropout);
  int used = -1;
  const int rc = launch_layernorm_bwd(a, (cudaStream_t)stream, &used);
  if (kernel_used) *kernel_used = used;
  return rc;
}

int univtg_op_head_final_bwd(const univtg_head_final_bwd* q, void* stream) {
  const char* fn = "univtg_op_head_final_bwd";
  UV_REQ(q != nullptr, "%s: null args", fn);
  UV_REQ(q->g_logits && q->g_spans && q->pred_logits && q->pred_spans && q->h_cls && q->h_span && q->w_cls && q->w_span && q->dz &&
             q->dh_cls && q->dh_span && q->gw_cls && q->gb_cls && q->gw_span && q->gb_span,
         "%s: null pointer argument", fn);
  UV_REQ((q->cs_cls == nullptr) == (q->cs_span == nullptr), "%s: cs_cls and cs_span must both be given or both be NULL", fn);
  UV_REQ(q->B >= 1 && q->Lv >= 1, "%s: B %d / Lv %d", fn, q->B, q->Lv);
  UV_REQ(q->d >= 8 && q->d % 8 == 0, "%s: d %d must be a positive multiple of 8 (128-bit loads)", fn, q->d);
  if (refuse_fmt2(q->fmt_act, fn) || refuse_fmt2(q->fmt_grad, fn)) return 1;
  UV_REQ((q->fmt_act == 0 || q->fmt_act == 1) && (q->fmt_grad == 0 || q->fmt_grad == 1), "%s: fmt_act / fmt_grad", fn);
  UV_REQ(al_(q->h_cls, 16) && al_(q->h_span, 16) && al_(q->dh_cls, 16) && al_(q->dh_span, 16) && al_(q->dz, 16) && al_(q->gw_cls, 16) &&
             al_(q->gw_span, 16) && al_(q->cs_cls, 16) && al_(q->cs_span, 16),
         "%s: h_*, dh_*, dz, gw_* and cs_* must be 16-byte aligned", fn);
  UV_REQ(al_(q->g_logits, 4) && al_(q->g_spans, 4) && al_(q->pred_logits, 4) && al_(q->pred_spans, 4) && al_(q->w_cls, 4) &&
             al_(q->w_span, 4) && al_(q->gb_cls, 4) && al_(q->gb_span, 4),
         "%s: misaligned fp32 pointer", fn);
  HeadFinalBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.g_logits = q->g_logits;
  a.g_spans = q->g_spans;
  a.pred_logits = q->pred_logits;
  a.pred_spans = q->pred_spans;
  a.h_cls = reinterpret_cast<const uint16_t*>(q->h_cls);
  a.h_span = reinterpret_cast<const uint16_t*>(q->h_span);
  a.w_cls = q->w_cls;
  a.w_span = q->w_span;
  a.dz = q->dz;
  a.dh_cls = reinterpret_cast<uint16_t*>(q->dh_cls);
  a.dh_span = reinterpret_cast<uint16_t*>(q->dh_span);
  a.gw_cls = q->gw_cls;
  a.gb_cls = q->gb_cls;
  a.gw_span = q->gw_span;
  a.gb_span = q->gb_span;
  a.cs_cls = q->cs_cls;
  a.cs_span = q->cs_span;
  a.in_scale = q->in_scale;
  a.pgrad_scale = q->pgrad_scale;
  a.B = q->B;
  a.Lv = q->Lv;
  a.d = q->d;
  a.fmt_act = q->fmt_act;
  a.fmt_grad = q->fmt_grad;
  return launch_head_final_bwd(a, (cudaStream_t)stream);
}

// text-row copy arguments shared by the two column-sum operators
static int txt_rows_arg(const char* fn, void* txt16, int L, int Lv, int txt_cols, int rows, int cols, int vec, TxtRows& t) {
  t = TxtRows{nullptr, 0, 0, 0};
  if (!txt16) return 0;
  UV_REQ(L >= 1 && Lv >= 0 && Lv < L && rows % L == 0, "%s: text rows need 0 <= Lv < L and rows %% L == 0 (L %d, Lv %d, rows %d)", fn, L,
         Lv, rows);
  UV_REQ(txt_cols >= vec && txt_cols <= cols && txt_cols % vec == 0, "%s: txt_cols %d must be a multiple of %d in [%d, cols]", fn, txt_cols,
         vec, vec);
  UV_REQ(al_(txt16, 2 * vec), "%s: txt16 must be %d-byte aligned", fn, 2 * vec);
  t = TxtRows{reinterpret_cast<uint16_t*>(txt16), L, Lv, txt_cols};
  return 0;
}

int univtg_op_colsum16(const void* in16, int32_t ld, int32_t rows, int32_t cols, int32_t fmt, float* colsum, float scale, void* txt16,
                       int32_t L, int32_t Lv, int32_t txt_cols, void* stream) {
  const char* fn = "univtg_op_colsum16";
  UV_REQ(in16 && colsum, "%s: null in16 or colsum", fn);
  UV_REQ(rows >= 1 && cols >= 8 && cols % 8 == 0 && ld >= cols && ld % 8 == 0, "%s: rows %d / cols %d / ld %d (multiples of 8, ld >= cols)", fn,
         rows, cols, ld);
  UV_REQ(al_(in16, 16) && al_(colsum, 16), "%s: in16 and colsum must be 16-byte aligned", fn);
  if (refuse_fmt2(fmt, fn)) return 1;
  UV_REQ(fmt == 0 || fmt == 1, "%s: fmt %d", fn, fmt);
  TxtRows t;
  if (txt_rows_arg(fn, txt16, L, Lv, txt_cols, rows, cols, 8, t)) return 1;
  return launch_colsum16(reinterpret_cast<const uint16_t*>(in16), ld, rows, cols, fmt, colsum, scale, (cudaStream_t)stream, t);
}

int univtg_op_cvt16_colsum(const float* in32, int32_t ld_in, void* out16, int32_t ld_out, int32_t rows, int32_t cols, int32_t fmt,
                           float* colsum, float colsum_scale, void* txt16, int32_t L, int32_t Lv, int32_t txt_cols, void* stream) {
  const char* fn = "univtg_op_cvt16_colsum";
  UV_REQ(in32 && out16, "%s: null in32 or out16", fn);
  UV_REQ(rows >= 1 && cols >= 4 && cols % 4 == 0 && ld_in >= cols && ld_in % 4 == 0 && ld_out >= cols && ld_out % 4 == 0,
         "%s: rows %d / cols %d / ld_in %d / ld_out %d (multiples of 4, pitches >= cols)", fn, rows, cols, ld_in, ld_out);
  UV_REQ(al_(in32, 16) && al_(out16, 8) && al_(colsum, 4), "%s: in32 must be 16-byte, out16 8-byte aligned", fn);
  if (refuse_fmt2(fmt, fn)) return 1;
  UV_REQ(fmt == 0 || fmt == 1, "%s: fmt %d", fn, fmt);
  TxtRows t;
  if (txt_rows_arg(fn, txt16, L, Lv, txt_cols, rows, cols, 4, t)) return 1;
  return launch_cvt16_colsum(in32, ld_in, reinterpret_cast<uint16_t*>(out16), ld_out, rows, cols, fmt, colsum, colsum_scale,
                             (cudaStream_t)stream, t);
}

int univtg_op_stream_gather(const float* dx, int32_t L, int32_t off, const float* extra, float extra_scale, void* out16, float* colsum,
                            float colsum_scale, int32_t B, int32_t Ls, int32_t d, int32_t fmt, void* stream) {
  const char* fn = "univtg_op_stream_gather";
  UV_REQ(dx && out16, "%s: null dx or out16", fn);
  UV_REQ(B >= 1 && Ls >= 1 && off >= 0 && off + Ls <= L, "%s: B %d / Ls %d / off %d / L %d (off + Ls <= L)", fn, B, Ls, off, L);
  UV_REQ(d >= 4 && d % 4 == 0, "%s: d %d must be a positive multiple of 4", fn, d);
  UV_REQ(al_(dx, 16) && al_(extra, 16) && al_(out16, 8) && al_(colsum, 4), "%s: dx / extra must be 16-byte, out16 8-byte aligned", fn);
  if (refuse_fmt2(fmt, fn)) return 1;
  UV_REQ(fmt == 0 || fmt == 1, "%s: fmt %d", fn, fmt);
  return launch_stream_gather(dx, L, off, extra, extra_scale, reinterpret_cast<uint16_t*>(out16), colsum, colsum_scale, B, Ls, d, fmt,
                              (cudaStream_t)stream);
}

int univtg_op_pool_bwd(const float* x_txt, const float* alpha, const float* w, const float* g_pooled, float* dx_txt, float* gw,
                       float out_scale, int32_t B, int32_t Lt, int32_t d, void* stream) {
  const char* fn = "univtg_op_pool_bwd";
  UV_REQ(x_txt && alpha && w && g_pooled && dx_txt && gw, "%s: null pointer argument", fn);
  UV_REQ(B >= 1 && d >= 1 && Lt >= 1 && (size_t)Lt * sizeof(float) <= 48 * 1024, "%s: B %d / Lt %d / d %d (Lt <= 12288)", fn, B, Lt, d);
  UV_REQ(al_(x_txt, 4) && al_(alpha, 4) && al_(w, 4) && al_(g_pooled, 4) && al_(dx_txt, 4) && al_(gw, 4), "%s: misaligned pointer", fn);
  PoolBwdArgs a;
  a.x_txt = x_txt;
  a.alpha = alpha;
  a.w = w;
  a.g_pooled = g_pooled;
  a.dx_txt = dx_txt;
  a.gw = gw;
  a.out_scale = out_scale;
  a.B = B;
  a.Lt = Lt;
  a.d = d;
  return launch_pool_bwd(a, (cudaStream_t)stream);
}

int univtg_op_txt_pos_bwd(const univtg_txt_pos_bwd* q, const univtg_rng* rng, int32_t mask_index, void* stream) {
  const char* fn = "univtg_op_txt_pos_bwd";
  UV_REQ(q != nullptr, "%s: null args", fn);
  UV_REQ(q->dpos && q->xt && q->table && q->gamma && q->mean && q->rstd && q->dx && q->dtable && q->dgamma && q->dbeta,
         "%s: null pointer argument", fn);
  UV_REQ(q->B >= 1 && q->Lt >= 1 && q->Lv >= 0 && q->Lv + q->Lt <= q->L, "%s: B %d / Lt %d / Lv %d / L %d (Lv + Lt <= L)", fn, q->B, q->Lt,
         q->Lv, q->L);
  UV_REQ(q->d >= 1 && q->d <= 1024, "%s: d %d (1..1024)", fn, q->d);
  UV_REQ(!rng || !(rng->input_dropout > 0.f) || mask_index >= 0, "%s: mask_index %d", fn, mask_index);
  TxtPosBwdArgs a;
  memset(&a, 0, sizeof(a));
  a.dpos = q->dpos;
  a.xt = q->xt;
  a.table = q->table;
  a.gamma = q->gamma;
  a.mean = q->mean;
  a.rstd = q->rstd;
  a.mul32 = q->mul32;
  if (!a.mul32 && rng && rng->input_dropout > 0.f) a.drop = make_drop_spec(rng->seed, (unsigned int)mask_index, rng->input_dropout);
  a.dx = q->dx;
  a.dtable = q->dtable;
  a.dgamma = q->dgamma;
  a.dbeta = q->dbeta;
  a.pgrad_scale = q->pgrad_scale;
  a.B = q->B;
  a.Lt = q->Lt;
  a.L = q->L;
  a.Lv = q->Lv;
  a.d = q->d;
  return launch_txt_pos_bwd(a, (cudaStream_t)stream);
}

int univtg_dropout_mask(const univtg_rng* rng, int32_t mask_index, size_t rows, size_t cols, float* out, void* stream) {
  if (!rng || !out || mask_index < 0 || cols == 0) {
    set_error("univtg_dropout_mask: bad argument");
    return 1;
  }
  return launch_dropout_mask(make_drop_spec(rng->seed, (unsigned int)mask_index, rng->input_dropout), rows * cols, cols, out,
                             (cudaStream_t)stream);
}

int univtg_attention_dropout_mask(const univtg_rng* rng, float p, int32_t layer, int32_t B, int32_t H, int32_t L, float* out,
                                  void* stream) {
  if (!rng || !out || layer < 0 || B < 1 || H < 1 || L < 1 || !(p >= 0.f && p < 1.f)) {
    set_error("univtg_attention_dropout_mask: bad argument (p must be in [0, 1))");
    return 1;
  }
  return launch_attention_dropout_mask(make_drop_spec(rng->seed, (unsigned int)layer, p), B, H, L, out, (cudaStream_t)stream);
}

uint64_t univtg_rng_seed_at(uint64_t base, uint64_t k) { return (uint64_t)rng_seed_at(base, k); }

int univtg_rng_advance(uint64_t base, uint64_t* counter_dev, uint64_t* seed_dev, void* stream) {
  const char* fn = "univtg_rng_advance";
  UV_REQ(counter_dev && seed_dev, "%s: null counter_dev or seed_dev", fn);
  UV_REQ(al_(counter_dev, 8) && al_(seed_dev, 8), "%s: counter_dev and seed_dev must be 8-byte aligned", fn);
  UV_REQ(counter_dev != seed_dev, "%s: counter_dev and seed_dev must be distinct", fn);
  return launch_rng_advance(base, reinterpret_cast<unsigned long long*>(counter_dev), reinterpret_cast<unsigned long long*>(seed_dev),
                            (cudaStream_t)stream);
}

int univtg_droppath_scales(const univtg_rng* rng, int32_t n_sites, int32_t batch, float* out, void* stream) {
  if (!rng || !out || n_sites < 1 || batch < 1) {
    set_error("univtg_droppath_scales: bad argument");
    return 1;
  }
  return launch_droppath_scales(rng->seed, n_sites * batch, 1.0f - rng->droppath, out, (cudaStream_t)stream);
}

size_t univtg_loss_scratch_bytes(int32_t B, int32_t Lv) { return make_loss_scratch(B, Lv, nullptr).total; }

namespace {
// What the criterion kernels (loss.cu) assume of their shapes: float4 rows (d % 4 == 0), at least one sample and one clip, and
// (Lv + 2B) floats of dynamic shared memory for loss_bwd_txt within the default 48 KiB.
bool loss_shape_ok(const char* fn, int32_t B, int32_t Lv, int32_t d) {
  if (B < 1 || Lv < 1 || d < 4 || d % 4 != 0 || (int64_t)B * Lv > INT32_MAX / 32) {
    set_error("%s: bad shape B %d, Lv %d, d %d (d must be a positive multiple of 4)", fn, B, Lv, d);
    return false;
  }
  if ((size_t)(Lv + 2 * B) * sizeof(float) > 48 * 1024 || B > 1536) {  // dynamic shared memory of loss_bwd_txt / loss_bwd_vid
    set_error("%s: B %d, Lv %d exceed the backward kernels' shared memory", fn, B, Lv);
    return false;
  }
  return true;
}

// the loss kernels read and write vid_mem_proj / txt_mem_proj rows and their gradients as float4
bool loss_aligned(const char* fn, const char* name, const void* p) {
  if (reinterpret_cast<uintptr_t>(p) % 16 != 0) {
    set_error("%s: %s must be 16-byte aligned", fn, name);
    return false;
  }
  return true;
}
}  // namespace

int univtg_loss_forward(const float* pred_logits, const float* pred_spans, const float* vid_mem_proj, const float* txt_mem_proj,
                        const float* timestamp, const float* timestamp_mask, const float* timestamp_window,
                        const float* span_labels_nn, const float* saliency_scores, const int64_t* saliency_pos_idx, int32_t B,
                        int32_t Lv, int32_t d, float eos_coef, float temperature, float* losses5, void* scratch, void* stream) {
  if (!pred_logits || !pred_spans || !vid_mem_proj || !txt_mem_proj || !timestamp_mask || !timestamp_window || !saliency_scores ||
      !losses5 || !scratch || ((timestamp == nullptr) != (span_labels_nn == nullptr))) {
    set_error("univtg_loss_forward: null argument");
    return 1;
  }
  const char* fn = "univtg_loss_forward";
  if (B > 256) {
    set_error("%s: batch %d > 256 not supported by the single-block reduction", fn, B);
    return 1;
  }
  if (!loss_shape_ok(fn, B, Lv, d) || !loss_aligned(fn, "vid_mem_proj", vid_mem_proj) ||
      !loss_aligned(fn, "txt_mem_proj", txt_mem_proj))
    return 1;
  const LossScratch s = make_loss_scratch(B, Lv, reinterpret_cast<uint8_t*>(scratch));
  LossArgs a;
  a.pred_logits = pred_logits;
  a.pred_spans = pred_spans;
  a.xv = vid_mem_proj;
  a.xt = txt_mem_proj;
  a.timestamp = timestamp;
  a.tmask = timestamp_mask;
  a.window = timestamp_window;
  a.span_gt = span_labels_nn;
  a.sal = saliency_scores;
  a.pos_idx = saliency_pos_idx;
  a.eos_coef = eos_coef;
  a.temperature = temperature;
  a.B = B;
  a.Lv = Lv;
  a.d = d;
  a.losses = losses5;
  a.g_spans_b = s.g_spans_b;
  a.g_spans_g = s.g_spans_g;
  a.g_logits_f = s.g_logits_f;
  a.cos_in = s.cos_in;
  a.vnorm = s.vnorm;
  a.tnorm = s.tnorm;
  a.sim = s.sim;
  a.g_cos_in = s.g_cos_in;
  a.g_sim = s.g_sim;
  return launch_loss_forward(a, (cudaStream_t)stream);
}

int univtg_loss_backward(const float* w5, const float* vid_mem_proj, const float* txt_mem_proj, const int64_t* saliency_pos_idx,
                         int32_t B, int32_t Lv, int32_t d, const void* scratch, float* d_logits, float* d_spans,
                         float* d_vid_mem_proj, float* d_txt_mem_proj, void* stream) {
  if (!w5 || !vid_mem_proj || !txt_mem_proj || !scratch || !d_logits || !d_spans || !d_vid_mem_proj || !d_txt_mem_proj) {
    set_error("univtg_loss_backward: null argument");
    return 1;
  }
  const char* fn = "univtg_loss_backward";
  if (B > 256) {
    set_error("%s: batch %d > 256 not supported by the single-block reduction", fn, B);
    return 1;
  }
  if (!loss_shape_ok(fn, B, Lv, d) || !loss_aligned(fn, "vid_mem_proj", vid_mem_proj) ||
      !loss_aligned(fn, "txt_mem_proj", txt_mem_proj) || !loss_aligned(fn, "d_vid_mem_proj", d_vid_mem_proj) ||
      !loss_aligned(fn, "d_txt_mem_proj", d_txt_mem_proj))
    return 1;
  const LossScratch s = make_loss_scratch(B, Lv, const_cast<uint8_t*>(reinterpret_cast<const uint8_t*>(scratch)));
  LossBwdArgs a;
  a.w = w5;
  a.g_spans_b = s.g_spans_b;
  a.g_spans_g = s.g_spans_g;
  a.g_logits_f = s.g_logits_f;
  a.cos_in = s.cos_in;
  a.vnorm = s.vnorm;
  a.tnorm = s.tnorm;
  a.sim = s.sim;
  a.g_cos_in = s.g_cos_in;
  a.g_sim = s.g_sim;
  a.xv = vid_mem_proj;
  a.xt = txt_mem_proj;
  a.pos_idx = saliency_pos_idx;
  a.B = B;
  a.Lv = Lv;
  a.d = d;
  a.d_logits = d_logits;
  a.d_spans = d_spans;
  a.d_xv = d_vid_mem_proj;
  a.d_xt = d_txt_mem_proj;
  return launch_loss_backward(a, (cudaStream_t)stream);
}

int univtg_qfvs_loss_forward(const float* pred_logits, const float* vid_mem_proj, const float* txt_mem_proj, const float* src_vid_mask,
                             const uint8_t* mask_gt, const float* saliency_scores, int32_t has_pos_labels, int32_t B, int32_t Lv,
                             int32_t d, float temperature, float* losses5, void* scratch, void* stream) {
  if (!pred_logits || !vid_mem_proj || !txt_mem_proj || !src_vid_mask || !mask_gt || !saliency_scores || !losses5 || !scratch) {
    set_error("univtg_qfvs_loss_forward: null argument");
    return 1;
  }
  const char* fn = "univtg_qfvs_loss_forward";
  if (!loss_shape_ok(fn, B, Lv, d) || !loss_aligned(fn, "vid_mem_proj", vid_mem_proj) ||
      !loss_aligned(fn, "txt_mem_proj", txt_mem_proj))
    return 1;
  const LossScratch s = make_loss_scratch(B, Lv, reinterpret_cast<uint8_t*>(scratch));
  QfvsLossArgs a;
  a.pred_logits = pred_logits;
  a.xv = vid_mem_proj;
  a.xt = txt_mem_proj;
  a.vmask = src_vid_mask;
  a.mask_gt = mask_gt;
  a.sal = saliency_scores;
  a.has_pos = has_pos_labels != 0;
  a.temperature = temperature;
  a.B = B;
  a.Lv = Lv;
  a.d = d;
  a.losses = losses5;
  a.g_spans_b = s.g_spans_b;
  a.g_spans_g = s.g_spans_g;
  a.g_logits_f = s.g_logits_f;
  a.cos_in = s.cos_in;
  a.vnorm = s.vnorm;
  a.tnorm = s.tnorm;
  a.g_cos_in = s.g_cos_in;
  return launch_qfvs_loss_forward(a, (cudaStream_t)stream);
}

int univtg_qfvs_loss_backward(const float* w5, const float* vid_mem_proj, const float* txt_mem_proj, int32_t B, int32_t Lv,
                              int32_t d, void* scratch, float* d_logits, float* d_vid_mem_proj, float* d_txt_mem_proj, void* stream) {
  if (!w5 || !vid_mem_proj || !txt_mem_proj || !scratch || !d_logits || !d_vid_mem_proj || !d_txt_mem_proj) {
    set_error("univtg_qfvs_loss_backward: null argument");
    return 1;
  }
  const char* fn = "univtg_qfvs_loss_backward";
  if (!loss_shape_ok(fn, B, Lv, d) || !loss_aligned(fn, "vid_mem_proj", vid_mem_proj) ||
      !loss_aligned(fn, "txt_mem_proj", txt_mem_proj) || !loss_aligned(fn, "d_vid_mem_proj", d_vid_mem_proj) ||
      !loss_aligned(fn, "d_txt_mem_proj", d_txt_mem_proj))
    return 1;
  const LossScratch s = make_loss_scratch(B, Lv, reinterpret_cast<uint8_t*>(scratch));
  LossBwdArgs a;
  a.w = w5;
  a.g_spans_b = s.g_spans_b;
  a.g_spans_g = s.g_spans_g;
  a.g_logits_f = s.g_logits_f;
  a.cos_in = s.cos_in;
  a.vnorm = s.vnorm;
  a.tnorm = s.tnorm;
  a.sim = s.sim;
  a.g_cos_in = s.g_cos_in;
  a.g_sim = s.g_sim;
  a.xv = vid_mem_proj;
  a.xt = txt_mem_proj;
  a.pos_idx = nullptr;
  a.B = B;
  a.Lv = Lv;
  a.d = d;
  a.d_logits = d_logits;
  a.d_spans = s.g_spans_b;  // pred_spans takes no part in the QFVS losses: loss_bwd_small's (zero) span gradient lands in scratch
  a.d_xv = d_vid_mem_proj;
  a.d_xt = d_txt_mem_proj;
  return launch_qfvs_loss_backward(a, (cudaStream_t)stream);
}

}  // extern "C"

#undef UV_REQ
