// SetCriterion of the reference for model_id = univtg (model/univtg.py:195-282, 338-351; utils/span_utils.py:46-122):
//   loss_b  smooth-L1 of (timestamp + pred_spans) vs span_labels_nn on foreground clips
//   loss_g  1 - generalised temporal IoU on foreground clips (only the diagonal of the reference's N x N matrix is used)
//   loss_f  weighted binary cross-entropy of pred_logits (foreground weight 1, valid background eos_coef)
//   loss_s_inter / loss_s_intra  two InfoNCE terms on cosine similarities (temperature 0.07)
// Forward computes the five losses AND the per-loss gradients w.r.t. the small model outputs; the backward kernel turns
// the cosine-matrix gradients into gradients of vid_mem_proj / txt_mem_proj for given loss weights.
#include <math.h>

#include "kernels.h"
#include "loss.h"
#include "ptx.cuh"

namespace uv {

// ------------------------------------------------------------------------------------------------
// kernel 1: cosines.  warps [0, B*Lv): cos_in[b,l] = cos(xv[b,l], xt[b]) and |xv[b,l]|;
//           warps [B*Lv, B*Lv + B*B): sim[b,b'] = cos(xv[b,pos_b], xt[b'])
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) loss_cos_kernel(const LossArgs a) {
  pdl_prologue();
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int n_in = a.B * a.Lv;
  if (gw >= n_in + a.B * a.B) return;
  int bv, lv, bt;
  if (gw < n_in) {
    bv = gw / a.Lv;
    lv = gw - bv * a.Lv;
    bt = bv;
  } else {
    const int k = gw - n_in;
    bv = k / a.B;
    bt = k - bv * a.B;
    lv = (int)a.pos_idx[bv];
  }
  const float* u = a.xv + ((size_t)bv * a.Lv + lv) * a.d;
  const float* v = a.xt + (size_t)bt * a.d;
  float dot = 0.f, nu = 0.f, nv = 0.f;
  for (int j = lane * 4; j < a.d; j += 128) {
    const float4 x = *reinterpret_cast<const float4*>(u + j);
    const float4 y = *reinterpret_cast<const float4*>(v + j);
    dot += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
    nu += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
    nv += y.x * y.x + y.y * y.y + y.z * y.z + y.w * y.w;
  }
  dot = warp_sum(dot);
  nu = warp_sum(nu);
  nv = warp_sum(nv);
  if (lane == 0) {
    const float un = fmaxf(sqrtf(nu), 1e-8f), vn = fmaxf(sqrtf(nv), 1e-8f);
    const float c = dot / (un * vn);
    if (gw < n_in) {
      a.cos_in[gw] = c;
      a.vnorm[gw] = un;
      if (lv == 0) a.tnorm[bv] = vn;
    } else {
      a.sim[gw - n_in] = c;
    }
  }
}

// block-wide sum of one float per thread (up to 1024 threads; s_red holds 32 floats)
__device__ __forceinline__ float block_sum(float v, float* s_red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  const int nw = blockDim.x >> 5;
  for (int i = 0; i < nw; ++i) t += s_red[i];
  return t;
}

// ------------------------------------------------------------------------------------------------
// kernel 2 (single block): all five losses + gradients w.r.t. pred_spans / pred_logits / cos_in / sim.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) loss_finish_kernel(const LossArgs a) {
  pdl_prologue();
  extern __shared__ float sm[];
  float* s_rowlse = sm;                // [B]   logsumexp over l of z[b, :]
  float* s_collse = s_rowlse + a.B;    // [B]   logsumexp over b' of z[b', pos_b]  (column pos_b)
  float* s_irow = s_collse + a.B;      // [B]   inter: logsumexp over b' of sim[b, b'] / tau
  float* s_icol = s_irow + a.B;        // [B]   inter: logsumexp over b of sim[b, b'] / tau
  int* s_pos = reinterpret_cast<int*>(s_icol + a.B);  // [B] positive clip index per sample
  __shared__ float s_red[32];
  const int tid = threadIdx.x, nt = blockDim.x;
  const int B = a.B, Lv = a.Lv, n = B * Lv;
  const float inv_tau = 1.0f / a.temperature;

  // ---- counts ----
  float c_fg = 0.f, c_valid = 0.f, c_sal = 0.f;
  for (int i = tid; i < n; i += nt) {
    c_fg += (a.window[i] != 0.f) ? 1.f : 0.f;
    c_valid += (a.tmask[i] != 0.f) ? 1.f : 0.f;
    c_sal += a.sal[i];
  }
  const float n_fg = block_sum(c_fg, s_red);
  const float n_valid = block_sum(c_valid, s_red);
  const float sal_sum = block_sum(c_sal, s_red);

  // ---- spans (loss_b, loss_g) and labels (loss_f) ----
  float lb = 0.f, lg = 0.f, lf = 0.f;
  for (int i = tid; i < n; i += nt) {
    const float w = a.window[i];
    const bool fg = w != 0.f;
    float gb0 = 0.f, gb1 = 0.f, gg0 = 0.f, gg1 = 0.f;
    // loss list without 'spans' (dset_type hl / vs, model/univtg.py:438-439): the targets carry no timestamp / span_labels_nn
    const bool spans = a.span_gt != nullptr && a.timestamp != nullptr;
    const float s1 = spans ? a.timestamp[2 * i] + a.pred_spans[2 * i] : 0.f;
    const float e1 = spans ? a.timestamp[2 * i + 1] + a.pred_spans[2 * i + 1] : 0.f;
    const float s2 = spans ? a.span_gt[2 * i] : 0.f, e2 = spans ? a.span_gt[2 * i + 1] : 0.f;
    if (spans) {  // smooth L1 (beta = 1) * window, normalised by the foreground count
      const float d0 = s1 - s2, d1 = e1 - e2;
      const float a0 = fabsf(d0), a1 = fabsf(d1);
      lb += ((a0 < 1.f ? 0.5f * d0 * d0 : a0 - 0.5f) + (a1 < 1.f ? 0.5f * d1 * d1 : a1 - 0.5f)) * w;
      gb0 = (a0 < 1.f ? d0 : (d0 > 0.f ? 1.f : -1.f)) * w / n_fg;
      gb1 = (a1 < 1.f ? d1 : (d1 > 0.f ? 1.f : -1.f)) * w / n_fg;
    }
    if (spans && fg) {  // generalised IoU of (s1, e1) vs (s2, e2)
      const float lo_i = fmaxf(s1, s2), hi_i = fminf(e1, e2);
      const float inter_raw = hi_i - lo_i;
      const float inter = fmaxf(inter_raw, 0.f);
      const float uni = (e1 - s1) + (e2 - s2) - inter;
      const float lo_e = fminf(s1, s2), hi_e = fmaxf(e1, e2);
      const float enc_raw = hi_e - lo_e;
      const float enc = fmaxf(enc_raw, 0.f);
      const float giou = inter / uni - (enc - uni) / enc;
      lg += 1.f - giou;
      // torch tie rules: max/min split evenly on ties; clamp(min=0) passes the gradient where x >= 0
      const float act_i = inter_raw >= 0.f ? 1.f : 0.f;
      const float dmax_s1 = s1 > s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);   // d max(s1,s2)/d s1
      const float dmin_e1 = e1 < e2 ? 1.f : (e1 == e2 ? 0.5f : 0.f);   // d min(e1,e2)/d e1
      const float di_s = -act_i * dmax_s1, di_e = act_i * dmin_e1;
      const float du_s = -1.f - di_s, du_e = 1.f - di_e;
      const float act_e = enc_raw >= 0.f ? 1.f : 0.f;
      const float dmin_s1 = s1 < s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
      const float dmax_e1 = e1 > e2 ? 1.f : (e1 == e2 ? 0.5f : 0.f);
      const float de_s = -act_e * dmin_s1, de_e = act_e * dmax_e1;
      // giou = inter/uni - 1 + uni/enc
      const float dg_s = (di_s * uni - inter * du_s) / (uni * uni) + (du_s * enc - uni * de_s) / (enc * enc);
      const float dg_e = (di_e * uni - inter * du_e) / (uni * uni) + (du_e * enc - uni * de_e) / (enc * enc);
      gg0 = -dg_s / n_fg;
      gg1 = -dg_e / n_fg;
    }
    a.g_spans_b[2 * i] = gb0;
    a.g_spans_b[2 * i + 1] = gb1;
    a.g_spans_g[2 * i] = gg0;
    a.g_spans_g[2 * i + 1] = gg1;
    {  // weighted BCE
      const float p = a.pred_logits[i];
      const bool valid = a.tmask[i] != 0.f;
      const float wt = fg ? 1.f : (valid ? a.eos_coef : 0.f);
      const float y = fg ? 1.f : 0.f;
      float gf = 0.f;
      if (valid) {
        const float lp = fmaxf(logf(p), -100.f), l1p = fmaxf(logf(1.f - p), -100.f);
        lf += -(y * lp + (1.f - y) * l1p) * wt;
        gf = wt * (p - y) / fmaxf(p * (1.f - p), 1e-12f);
      }
      // the reference's (bce * mask).sum() / mask.sum(): 0 at masked clips, NaN everywhere (0 / 0) without any valid clip
      a.g_logits_f[i] = gf / n_valid;
    }
  }
  lb = block_sum(lb, s_red);
  lg = block_sum(lg, s_red);
  lf = block_sum(lf, s_red);
  if (tid == 0) {
    const bool spans = a.span_gt != nullptr && a.timestamp != nullptr;
    a.losses[0] = spans ? lb / n_fg : 0.f;
    a.losses[1] = spans ? lg / n_fg : 0.f;
    a.losses[2] = lf / n_valid;
  }

  // ---- saliency ----
  if (a.pos_idx == nullptr || sal_sum == 0.f) {  // reference returns 0. for both terms
    for (int i = tid; i < n; i += nt) a.g_cos_in[i] = 0.f;
    for (int i = tid; i < B * B; i += nt) a.g_sim[i] = 0.f;
    if (tid == 0) {
      a.losses[3] = 0.f;
      a.losses[4] = 0.f;
    }
    return;
  }
  for (int b = tid; b < B; b += nt) s_pos[b] = (int)a.pos_idx[b];
  const int warp = tid >> 5, lane = tid & 31, nwarps = nt >> 5;
  // inter-video: sim [B, B]; one warp per row / column
  for (int r = warp; r < 2 * B; r += nwarps) {
    const int b = r % B;
    const bool col = r >= B;
    float mx = -INFINITY;
    for (int k = lane; k < B; k += 32) mx = fmaxf(mx, (col ? a.sim[k * B + b] : a.sim[b * B + k]) * inv_tau);
    mx = warp_max(mx);
    float s = 0.f;
    for (int k = lane; k < B; k += 32) s += expf((col ? a.sim[k * B + b] : a.sim[b * B + k]) * inv_tau - mx);
    s = warp_sum(s);
    if (lane == 0) (col ? s_icol : s_irow)[b] = mx + logf(s);
  }
  __syncthreads();
  float l_inter = 0.f;
  for (int b = tid; b < B; b += nt) l_inter += 2.f * a.sim[b * B + b] * inv_tau - s_irow[b] - s_icol[b];
  l_inter = block_sum(l_inter, s_red);
  for (int i = tid; i < B * B; i += nt) {
    const int b = i / B, k = i - b * B;
    const float z = a.sim[i] * inv_tau;
    const float dlt = (b == k) ? 2.f : 0.f;
    a.g_sim[i] = -(dlt - expf(z - s_irow[b]) - expf(z - s_icol[k])) * inv_tau / (float)B;
  }
  // intra-video: z[b,l] = (cos_in[b,l] + log(keep + 1e-45)) / tau
  //   keep[b,l] = ((sal[b,l] < sal[b,pos_b]) or l == pos_b) and tmask[b,l]
  auto zval = [&](int b, int l) -> float {
    const int p = s_pos[b];
    const bool keep = ((a.sal[b * Lv + l] < a.sal[b * Lv + p]) || (l == p)) && (a.tmask[b * Lv + l] != 0.f);
    return (a.cos_in[b * Lv + l] + logf((keep ? 1.f : 0.f) + 1e-45f)) * inv_tau;
  };
  for (int r = warp; r < 2 * B; r += nwarps) {
    const int b = r % B;
    const bool col = r >= B;  // row b: over clips l; column pos_b: over samples b'
    const int p = s_pos[b];
    const int cnt = col ? B : Lv;
    float mx = -INFINITY;
    for (int k = lane; k < cnt; k += 32) mx = fmaxf(mx, col ? zval(k, p) : zval(b, k));
    mx = warp_max(mx);
    float s = 0.f;
    for (int k = lane; k < cnt; k += 32) s += expf((col ? zval(k, p) : zval(b, k)) - mx);
    s = warp_sum(s);
    if (lane == 0) (col ? s_collse : s_rowlse)[b] = mx + logf(s);
  }
  __syncthreads();
  float l_intra = 0.f;
  for (int b = tid; b < B; b += nt) {
    const float zp = zval(b, s_pos[b]);
    l_intra += 2.f * zp - s_rowlse[b] - s_collse[b];
  }
  l_intra = block_sum(l_intra, s_red);
  for (int i = tid; i < n; i += nt) {
    const int b = i / Lv, l = i - b * Lv;
    const float z = zval(b, l);
    // d/dz[b,l] of -(1/B) sum_b'' [ z[b'',p''] - rowlse[b''] + z[b'',p''] - collse(p'')[b''] ]
    float g = -expf(z - s_rowlse[b]);
    if (l == s_pos[b]) g += 2.f;
    for (int k = 0; k < B; ++k)
      if (s_pos[k] == l) g -= expf(z - s_collse[k]);
    a.g_cos_in[i] = -g * inv_tau / (float)B;
  }
  if (tid == 0) {
    a.losses[3] = -l_inter / (float)B;
    a.losses[4] = -l_intra / (float)B;
  }
}

int launch_loss_forward(const LossArgs& a, cudaStream_t stream) {
  if (a.pos_idx != nullptr) {
    const int warps = a.B * a.Lv + a.B * a.B;
    launch_k(loss_cos_kernel, dim3((warps * 32 + 255) / 256), dim3(256), 0, stream, a);
  }
  launch_k(loss_finish_kernel, dim3(1), dim3(1024), (size_t)5 * a.B * sizeof(float), stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("loss forward launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// QFVS criterion (reference model/univtg_qfvs.py:215-261, 358-377), one block, any N = B * Lv.
//   kept positions: i with mask_gt[i]; the k-th kept position (k = exclusive prefix count of mask_gt) pairs with t = sal[k]
//   loss_f        sum over kept of BCE(pred_logits, t) (log clamped at -100) / sum(t)
//   loss_s_intra  -mean over kept positions with t > 0 of log softmax(z), the softmax over all kept positions
//   z[i] = (cos_in[i] + log(vmask[i] + 1e-45)) / tau: the model's saliency_scores / tau
// Both are 0 when sum(t) == 0, loss_s_intra also without saliency_pos_labels; their gradients are then exactly 0.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_max(float v, float* s_red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
  const int nw = blockDim.x >> 5;
  for (int i = 0; i < nw; ++i) t = fmaxf(t, s_red[i]);
  return t;
}

__global__ void __launch_bounds__(1024) qfvs_loss_kernel(const QfvsLossArgs a) {
  pdl_prologue();
  __shared__ float s_red[32];
  __shared__ int s_cnt[32];
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
  const int n = a.B * a.Lv;
  const float inv_tau = 1.0f / a.temperature;
  // pass 1, in chunks of nt positions: ranks, target sum, positive count, BCE sum, sum of z over positives and a running
  // (max, sum of exp) of z per thread.  Each thread parks t (0 when not kept) in g_logits_f[i] and the keep flag in g_cos_in[i]
  // for pass 2, which visits the same i with the same thread.
  int ranked = 0;  // kept positions in earlier chunks
  float c_t = 0.f, c_pos = 0.f, c_bce = 0.f, c_zpos = 0.f, mx = -INFINITY, se = 0.f;
  for (int base = 0; base < n; base += nt) {
    const int i = base + tid;
    const bool keep = i < n && a.mask_gt[i] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_cnt[warp] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < nw; ++w) {
      const int c = s_cnt[w];
      before += w < warp ? c : 0;
      total += c;
    }
    __syncthreads();  // s_cnt is rewritten by the next chunk
    if (i < n) {
      float t = 0.f;
      if (keep) {
        t = a.sal[ranked + before + __popc(bal & ((1u << lane) - 1u))];
        const float p = a.pred_logits[i];
        const float lp = fmaxf(logf(p), -100.f), l1p = fmaxf(logf(1.f - p), -100.f);
        c_t += t;
        c_bce += -(t * lp + (1.f - t) * l1p);
        const float z = (a.cos_in[i] + logf(a.vmask[i] + 1e-45f)) * inv_tau;
        if (t > 0.f) {
          c_pos += 1.f;
          c_zpos += z;
        }
        if (z > mx) {
          se = se * expf(mx - z) + 1.f;
          mx = z;
        } else {
          se += expf(z - mx);
        }
      }
      a.g_logits_f[i] = t;
      a.g_cos_in[i] = keep ? 1.f : 0.f;
    }
    ranked += total;
  }
  const float sum_t = block_sum(c_t, s_red);
  const float n_pos = block_sum(c_pos, s_red);
  const float bce = block_sum(c_bce, s_red);
  const float zpos = block_sum(c_zpos, s_red);
  const float zmax = block_max(mx, s_red);
  const float lse = zmax + logf(block_sum(mx == -INFINITY ? 0.f : se * expf(mx - zmax), s_red));
  const bool on = sum_t != 0.f;          // reference: `if saliency_scores.sum() == 0: return 0.`
  const bool sal_on = on && a.has_pos != 0;
  // pass 2: unit gradients d loss_f / d pred_logits (torch's BCE backward) and d loss_s_intra / d cos_in
  for (int i = tid; i < n; i += nt) {
    const float t = a.g_logits_f[i];
    const bool keep = a.g_cos_in[i] != 0.f;
    float gf = 0.f, gc = 0.f;
    if (keep && on) {
      const float p = a.pred_logits[i];
      gf = (p - t) / fmaxf(p * (1.f - p), 1e-12f) / sum_t;
    }
    if (keep && sal_on) {
      const float z = (a.cos_in[i] + logf(a.vmask[i] + 1e-45f)) * inv_tau;
      gc = (expf(z - lse) - (t > 0.f ? 1.f / n_pos : 0.f)) * inv_tau;
    }
    a.g_logits_f[i] = gf;
    a.g_cos_in[i] = gc;
    a.g_spans_b[2 * i] = 0.f;
    a.g_spans_b[2 * i + 1] = 0.f;
    a.g_spans_g[2 * i] = 0.f;
    a.g_spans_g[2 * i + 1] = 0.f;
  }
  if (tid == 0) {
    a.losses[0] = 0.f;
    a.losses[1] = 0.f;
    a.losses[2] = on ? bce / sum_t : 0.f;
    a.losses[3] = 0.f;
    a.losses[4] = sal_on ? lse - zpos / n_pos : 0.f;
  }
}

int launch_qfvs_loss_forward(const QfvsLossArgs& q, cudaStream_t stream) {
  // cosines through loss_cos_kernel with one warp per block: every warp index is below B * Lv, so its B x B part never runs
  LossArgs c = {};
  c.xv = q.xv;
  c.xt = q.xt;
  c.B = q.B;
  c.Lv = q.Lv;
  c.d = q.d;
  c.cos_in = q.cos_in;
  c.vnorm = q.vnorm;
  c.tnorm = q.tnorm;
  launch_k(loss_cos_kernel, dim3(q.B * q.Lv), dim3(32), 0, stream, c);
  launch_k(qfvs_loss_kernel, dim3(1), dim3(1024), 0, stream, q);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("qfvs loss forward launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

// ------------------------------------------------------------------------------------------------
// backward: weights w[5] (dL/d loss_k) -> gradients of the model outputs.
//   d cos(u, v)/du = v / (|u||v|) - cos * u / |u|^2
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) loss_bwd_small_kernel(const LossBwdArgs a) {
  pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = a.B * a.Lv;
  if (i >= n) return;
  const float wb = a.w[0], wg = a.w[1], wf = a.w[2];
  a.d_logits[i] = wf * a.g_logits_f[i];
  a.d_spans[2 * i] = wb * a.g_spans_b[2 * i] + wg * a.g_spans_g[2 * i];
  a.d_spans[2 * i + 1] = wb * a.g_spans_b[2 * i + 1] + wg * a.g_spans_g[2 * i + 1];
}

// one warp per (b, l): d xv[b, l, :]
__global__ void __launch_bounds__(256) loss_bwd_vid_kernel(const LossBwdArgs a) {
  pdl_prologue();
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= a.B * a.Lv) return;
  const int b = gw / a.Lv, l = gw - b * a.Lv;
  const float w_inter = a.w[3], w_intra = a.w[4];
  const float un = a.vnorm[gw];
  const float gi = w_intra * a.g_cos_in[gw];
  const float ci = a.cos_in[gw];
  const bool is_pos = a.pos_idx != nullptr && (int)a.pos_idx[b] == l;
  const float* u = a.xv + (size_t)gw * a.d;
  float* out = a.d_xv + (size_t)gw * a.d;
  extern __shared__ float s_c1[];  // [8 warps][B] coefficients of xt[k] for the positive row of a sample
  float* c1w = s_c1 + (size_t)(threadIdx.x >> 5) * a.B;
  const float s1 = gi / (un * a.tnorm[b]);
  float s2 = gi * ci / (un * un);
  if (is_pos) {
    float s2p = 0.f;
    for (int k = lane; k < a.B; k += 32) {
      const float gx = w_inter * a.g_sim[b * a.B + k];
      c1w[k] = gx / (un * a.tnorm[k]);
      s2p += gx * a.sim[b * a.B + k] / (un * un);
    }
    s2 += warp_sum(s2p);
    __syncwarp();
  }
  for (int j = lane * 4; j < a.d; j += 128) {
    const float4 x = *reinterpret_cast<const float4*>(u + j);
    const float4 t = *reinterpret_cast<const float4*>(a.xt + (size_t)b * a.d + j);
    float4 o = make_float4(s1 * t.x, s1 * t.y, s1 * t.z, s1 * t.w);
    if (is_pos) {
#pragma unroll 4
      for (int k = 0; k < a.B; ++k) {
        const float4 tk = *reinterpret_cast<const float4*>(a.xt + (size_t)k * a.d + j);
        const float c1 = c1w[k];
        o.x += c1 * tk.x;
        o.y += c1 * tk.y;
        o.z += c1 * tk.z;
        o.w += c1 * tk.w;
      }
    }
    o.x -= s2 * x.x;
    o.y -= s2 * x.y;
    o.z -= s2 * x.z;
    o.w -= s2 * x.w;
    *reinterpret_cast<float4*>(out + j) = o;
  }
}

// one block per (sample b, 128-column chunk): d xt[b, :].  The per-row scalar factors are staged in shared memory first so
// the column loop is one coalesced load + FMA per contributing clip row.
__global__ void __launch_bounds__(128) loss_bwd_txt_kernel(const LossBwdArgs a) {
  pdl_prologue();
  extern __shared__ float s_coef[];                          // [Lv + B] factor of xv[row] in d xt[b]
  int* s_row = reinterpret_cast<int*>(s_coef + a.Lv + a.B);  // [B] clip row of the positive of sample k
  __shared__ float s_red[4];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float w_inter = a.w[3], w_intra = a.w[4];
  const float tn = a.tnorm[b];
  float part = 0.f;  // sum of g * cos: factor of -xt[b] / |xt[b]|^2
  for (int l = tid; l < a.Lv; l += 128) {  // vnorm and tnorm are clamped >= 1e-8 by the forward
    const int i = b * a.Lv + l;
    const float g = w_intra * a.g_cos_in[i];
    s_coef[l] = g / (a.vnorm[i] * tn);
    part += g * a.cos_in[i];
  }
  const int nk = a.pos_idx != nullptr ? a.B : 0;
  for (int k = tid; k < nk; k += 128) {
    const float g = w_inter * a.g_sim[k * a.B + b];
    const int i = k * a.Lv + (int)a.pos_idx[k];
    s_coef[a.Lv + k] = g / (a.vnorm[i] * tn);
    s_row[k] = i;
    part += g * a.sim[k * a.B + b];
  }
  part = warp_sum(part);
  if ((tid & 31) == 0) s_red[tid >> 5] = part;
  __syncthreads();
  const float c2 = (s_red[0] + s_red[1] + s_red[2] + s_red[3]) / (tn * tn);
  for (int j = blockIdx.y * 128 + tid; j < a.d; j += gridDim.y * 128) {
    float o = -c2 * a.xt[(size_t)b * a.d + j];
    const float* xv = a.xv + (size_t)b * a.Lv * a.d + j;
#pragma unroll 8
    for (int l = 0; l < a.Lv; ++l) o += s_coef[l] * xv[(size_t)l * a.d];
#pragma unroll 4
    for (int k = 0; k < nk; ++k) o += s_coef[a.Lv + k] * a.xv[(size_t)s_row[k] * a.d + j];
    a.d_xt[(size_t)b * a.d + j] = o;
  }
}

int launch_loss_backward(const LossBwdArgs& a, cudaStream_t stream) {
  const int n = a.B * a.Lv;
  launch_k(loss_bwd_small_kernel, dim3((n + 255) / 256), dim3(256), 0, stream, a);
  if (a.pos_idx == nullptr) {
    // targets without saliency_pos_labels: the reference returns the constant 0. for both saliency losses
    // (model/univtg.py:236-237), so nothing flows into vid_mem_proj / txt_mem_proj; the forward skipped loss_cos_kernel and
    // the cosine scratch is unwritten - do not read it.
    cudaMemsetAsync(a.d_xv, 0, (size_t)n * a.d * sizeof(float), stream);
    cudaMemsetAsync(a.d_xt, 0, (size_t)a.B * a.d * sizeof(float), stream);
    cudaError_t e0 = cudaGetLastError();
    if (e0 != cudaSuccess) set_error("loss backward launch failed: %s", cudaGetErrorString(e0));
    return (int)e0;
  }
  launch_k(loss_bwd_vid_kernel, dim3((n * 32 + 255) / 256), dim3(256), (size_t)8 * a.B * sizeof(float), stream, a);
  launch_k(loss_bwd_txt_kernel, dim3(a.B, (a.d + 127) / 128), dim3(128), (size_t)(a.Lv + 2 * a.B) * sizeof(float), stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("loss backward launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

int launch_qfvs_loss_backward(const LossBwdArgs& a, cudaStream_t stream) {
  const int n = a.B * a.Lv;
  launch_k(loss_bwd_small_kernel, dim3((n + 255) / 256), dim3(256), 0, stream, a);
  launch_k(loss_bwd_vid_kernel, dim3((n * 32 + 255) / 256), dim3(256), (size_t)8 * a.B * sizeof(float), stream, a);
  launch_k(loss_bwd_txt_kernel, dim3(a.B, (a.d + 127) / 128), dim3(128), (size_t)(a.Lv + 2 * a.B) * sizeof(float), stream, a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("qfvs loss backward launch failed: %s", cudaGetErrorString(e));
  return (int)e;
}

}  // namespace uv
