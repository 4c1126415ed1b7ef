// CLIP feature extraction (include/univtg_b200.h, univtg_clip_*): the ViT image tower and the text tower of OpenAI CLIP
// (reference run_on_video/clip/model.py), inference only.
//
// Both towers are pre-norm transformers over an fp32 residual stream x (ResidualAttentionBlock.forward, model.py:185-188):
//   a16 = LN_1(x);  qkv = a16 W_in^T + b  (GEMM, 16-bit out);  o = attention(qkv)  (dh = 64 wgmma kernel; causal for text);
//   x += o W_out^T + b        (GEMM, residual epilogue into x);
//   a16 = LN_2(x);  h = QuickGELU(a16 W_fc^T + b)  (GEMM epilogue);  x += h W_proj^T + b  (GEMM, residual epilogue)
// Front ends and heads are row kernels of this file; the GEMMs, the attention kernel and the LayerNorm kernel are the library's.
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <climits>
#include <vector>

#include <cuda_fp16.h>

#include "plan.h"
#include "ptx.cuh"

namespace {

constexpr int kClipMaxLayers = 64;
constexpr int kClipMaxWidth = 1024;  // warp-per-row kernels hold a row in registers: 32 values per lane

struct ClipBlockPk {
  size_t w_in, b_in, w_out, b_out, ln1w, ln1b, w_fc, b_fc, w_pr, b_pr, ln2w, ln2b;
};
struct ClipPacked {
  // vision
  size_t conv16;          // 16-bit [Wv, kpad]: conv1.weight flattened in (c, ky, kx) order, K zero-padded to 64
  size_t cls, vpos;       // fp32 [Wv], [Lp, Wv]
  size_t ln_pre_w, ln_pre_b, ln_post_w, ln_post_b;
  size_t vproj16;         // 16-bit [E, Wv] = visual.proj^T
  ClipBlockPk vblk[kClipMaxLayers];
  // text
  size_t tok, tpos;       // fp32 [V, Wt], [C, Wt]
  size_t ln_f_w, ln_f_b;
  size_t tproj16;         // 16-bit [E, Wt] = text_projection^T
  ClipBlockPk tblk[kClipMaxLayers];
  size_t total;
};

struct ClipShape {
  int grid, pc, lp, kpad;  // patches per side, patches per frame, tokens per frame (pc + 1), padded K of the patch GEMM
};
inline ClipShape clip_shape(const univtg_clip_config& c) {
  ClipShape s;
  s.grid = c.image_resolution / c.patch_size;
  s.pc = s.grid * s.grid;
  s.lp = s.pc + 1;
  s.kpad = pad64(3 * c.patch_size * c.patch_size);
  return s;
}

bool clip_check_cfg(const univtg_clip_config* c, const char* fn) {
  if (!c) {
    set_error("%s: cfg is null", fn);
    return false;
  }
  if (c->operand_format == 2) {
    set_error("%s: operand_format 2 (fp16x3) is not supported by the CLIP encoder; use 0 (fp16) or 1 (bf16)", fn);
    return false;
  }
#define CLIP_REQ(cond, ...)  \
  if (!(cond)) {             \
    set_error(__VA_ARGS__);  \
    return false;            \
  }
  CLIP_REQ(c->operand_format == 0 || c->operand_format == 1, "%s: cfg->operand_format %d must be 0 (fp16) or 1 (bf16)", fn,
           c->operand_format);
  CLIP_REQ(c->vision_width > 0 && c->vision_width % 64 == 0 && c->vision_width <= kClipMaxWidth,
           "%s: cfg->vision_width %d must be a positive multiple of 64 (heads are 64 wide) and <= %d", fn, c->vision_width, kClipMaxWidth);
  CLIP_REQ(c->text_width > 0 && c->text_width % 64 == 0 && c->text_width <= kClipMaxWidth,
           "%s: cfg->text_width %d must be a positive multiple of 64 (heads are 64 wide) and <= %d", fn, c->text_width, kClipMaxWidth);
  CLIP_REQ(c->vision_layers >= 1 && c->vision_layers <= kClipMaxLayers, "%s: cfg->vision_layers %d out of range [1, %d]", fn,
           c->vision_layers, kClipMaxLayers);
  CLIP_REQ(c->text_layers >= 1 && c->text_layers <= kClipMaxLayers, "%s: cfg->text_layers %d out of range [1, %d]", fn, c->text_layers,
           kClipMaxLayers);
  CLIP_REQ(c->patch_size >= 1 && c->image_resolution >= c->patch_size && c->image_resolution % c->patch_size == 0,
           "%s: cfg->image_resolution %d must be a positive multiple of cfg->patch_size %d", fn, c->image_resolution, c->patch_size);
  CLIP_REQ(c->embed_dim > 0 && c->embed_dim % 16 == 0, "%s: cfg->embed_dim %d must be a positive multiple of 16", fn, c->embed_dim);
  CLIP_REQ(c->context_length >= 1, "%s: cfg->context_length %d must be positive", fn, c->context_length);
  CLIP_REQ(c->vocab_size >= 1, "%s: cfg->vocab_size %d must be positive", fn, c->vocab_size);
#undef CLIP_REQ
  return true;
}

void clip_blocks_layout(Cursor& cur, ClipBlockPk* blk, int layers, size_t W) {
  for (int l = 0; l < layers; ++l) {
    ClipBlockPk& b = blk[l];
    b.w_in = cur.take(3 * W * W * 2);
    b.b_in = cur.take(3 * W * 4);
    b.w_out = cur.take(W * W * 2);
    b.b_out = cur.take(W * 4);
    b.ln1w = cur.take(W * 4);
    b.ln1b = cur.take(W * 4);
    b.w_fc = cur.take(4 * W * W * 2);
    b.b_fc = cur.take(4 * W * 4);
    b.w_pr = cur.take(4 * W * W * 2);
    b.b_pr = cur.take(W * 4);
    b.ln2w = cur.take(W * 4);
    b.ln2b = cur.take(W * 4);
  }
}

ClipPacked clip_layout(const univtg_clip_config& c) {
  ClipPacked P;
  memset(&P, 0, sizeof(P));
  const ClipShape s = clip_shape(c);
  const size_t Wv = c.vision_width, Wt = c.text_width, E = c.embed_dim;
  Cursor cur;
  P.conv16 = cur.take(Wv * s.kpad * 2);
  P.cls = cur.take(Wv * 4);
  P.vpos = cur.take((size_t)s.lp * Wv * 4);
  P.ln_pre_w = cur.take(Wv * 4);
  P.ln_pre_b = cur.take(Wv * 4);
  clip_blocks_layout(cur, P.vblk, c.vision_layers, Wv);
  P.ln_post_w = cur.take(Wv * 4);
  P.ln_post_b = cur.take(Wv * 4);
  P.vproj16 = cur.take(E * Wv * 2);
  P.tok = cur.take((size_t)c.vocab_size * Wt * 4);
  P.tpos = cur.take((size_t)c.context_length * Wt * 4);
  clip_blocks_layout(cur, P.tblk, c.text_layers, Wt);
  P.ln_f_w = cur.take(Wt * 4);
  P.ln_f_b = cur.take(Wt * 4);
  P.tproj16 = cur.take(E * Wt * 2);
  P.total = cur.off;
  return P;
}

// Buffers of one tower's forward over M = sequences x tokens rows of width W.
struct ClipWs {
  uint16_t* patch16;  // vision: [T * pc, kpad] A operand of the patch embedding
  float* x32;         // [M, W] residual stream
  uint16_t *a16, *qkv16, *attn16, *h16;  // [M, W], [M, 3W], [M, W], [M, 4W]
  float* ones;        // [M] key mask: every key valid
  uint16_t* head16;   // [sequences, W] LayerNorm'd class / EOT rows (A operand of the projection)
  size_t total;
};
ClipWs clip_ws(size_t M, size_t W, size_t seqs, size_t patch_elems, uint8_t* base) {
  ClipWs w;
  memset(&w, 0, sizeof(w));
  Cursor cur;
  auto take16 = [&](size_t e) { return reinterpret_cast<uint16_t*>(base + cur.take(e * 2)); };
  auto take32 = [&](size_t e) { return reinterpret_cast<float*>(base + cur.take(e * 4)); };
  if (patch_elems) w.patch16 = take16(patch_elems);
  w.x32 = take32(M * W);
  w.a16 = take16(M * W);
  w.qkv16 = take16(M * 3 * W);
  w.attn16 = take16(M * W);
  w.h16 = take16(M * 4 * W);
  w.ones = take32(M);
  w.head16 = take16(seqs * W);
  w.total = cur.off;
  return w;
}
size_t clip_vision_ws_bytes(const univtg_clip_config& c, size_t T) {
  if (T == 0) return 0;
  const ClipShape s = clip_shape(c);
  return clip_ws(T * s.lp, c.vision_width, T, T * s.pc * s.kpad, nullptr).total;
}
size_t clip_text_ws_bytes(const univtg_clip_config& c, size_t N, size_t Lc) {
  if (N == 0 || Lc == 0) return 0;
  return clip_ws(N * Lc, c.text_width, N, 0, nullptr).total;
}

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float clip_src(const void* p, size_t i, int dt) {
  return dt == 0 ? reinterpret_cast<const float*>(p)[i] : __half2float(reinterpret_cast<const __half*>(p)[i]);
}

// kind 0: [rows, cols] -> 16-bit [rows, ld] (columns >= cols zero); 1: fp32 copy of rows * cols; 2: 16-bit transpose -> [cols, rows]
__global__ void __launch_bounds__(256) clip_pack_kernel(const void* src, int dt, void* dst, int kind, int rows, int cols, int ld,
                                                        int fmt) {
  pdl_prologue();
  const size_t n = kind == 0 ? (size_t)rows * ld : (size_t)rows * cols;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (kind == 0) {
      const int r = (int)(i / ld), c = (int)(i % ld);
      reinterpret_cast<uint16_t*>(dst)[i] = cvt16(c < cols ? clip_src(src, (size_t)r * cols + c, dt) : 0.f, fmt);
    } else if (kind == 1) {
      reinterpret_cast<float*>(dst)[i] = clip_src(src, i, dt);
    } else {
      const int c = (int)(i / rows), r = (int)(i % rows);  // destination [cols, rows]
      reinterpret_cast<uint16_t*>(dst)[i] = cvt16(clip_src(src, (size_t)r * cols + c, dt), fmt);
    }
  }
}

// Frames -> A operand of the patch embedding: row t * pc + py * grid + px, column k = c * P^2 + ky * P + kx (conv1.weight's
// order), columns >= 3 P^2 zero.  kind 0: uint8 [T, R, R, 3] with Preprocessing (run_on_video/preprocessing.py:4-25) in fp32;
// kind 1: normalised f32 [T, 3, R, R].
__global__ void __launch_bounds__(256) clip_frames_kernel(const void* pixels, int kind, int T, int R, int P, int grid, int kpad,
                                                          int fmt, uint16_t* __restrict__ out) {
  pdl_prologue();
  const int K = 3 * P * P, pc = grid * grid;
  const size_t n = (size_t)T * pc * kpad;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % kpad);
    const size_t row = i / kpad;
    float v = 0.f;
    if (k < K) {
      const int t = (int)(row / pc), p = (int)(row % pc);
      const int c = k / (P * P), ky = (k / P) % P, kx = k % P;
      const int y = (p / grid) * P + ky, x = (p % grid) * P + kx;
      if (kind == 0) {
        const float mean = c == 0 ? 0.48145466f : c == 1 ? 0.4578275f : 0.40821073f;
        const float sd = c == 0 ? 0.26862954f : c == 1 ? 0.26130258f : 0.27577711f;
        const float u = (float)reinterpret_cast<const uint8_t*>(pixels)[(((size_t)t * R + y) * R + x) * 3 + c];
        v = (u / 255.0f - mean) / (sd + 1e-8f);
      } else {
        v = reinterpret_cast<const float*>(pixels)[(((size_t)t * 3 + c) * R + y) * R + x];
      }
    }
    out[i] = cvt16(v, fmt);
  }
}

// LayerNorm of the W values a lane holds (columns lane + 32 i), eps 1e-5, biased variance.
__device__ __forceinline__ void clip_ln(float (&v)[kClipMaxWidth / 32], int W, const float* __restrict__ g, const float* __restrict__ b,
                                        int lane, float (&y)[kClipMaxWidth / 32]) {
  const int nv = W >> 5;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kClipMaxWidth / 32; ++i)
    if (i < nv) s += v[i];
  const float mean = warp_sum(s) / (float)W;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kClipMaxWidth / 32; ++i)
    if (i < nv) q += (v[i] - mean) * (v[i] - mean);
  const float rstd = rsqrtf(warp_sum(q) / (float)W + 1e-5f);
#pragma unroll
  for (int i = 0; i < kClipMaxWidth / 32; ++i)
    if (i < nv) y[i] = (v[i] - mean) * rstd * __ldg(g + lane + 32 * i) + __ldg(b + lane + 32 * i);
}

// Embedding row kernel, one warp per stream row r = s * L + l (a warp-stride loop: the grid may hold fewer warps than rows):
//   vision (tokens == null): v = (l == 0 ? class_embedding : x32[r]) + pos[l];  x = ln_pre(v)
//   text: v = token_embedding[tokens[s * ctx + l]] + pos[l];  x = v
// then x32[r] = x, a16[r] = 16-bit(ln_1 of block 0 (x)), ones[r] = 1.
__global__ void __launch_bounds__(256) clip_embed_kernel(float* __restrict__ x32, const float* __restrict__ cls,
                                                         const int64_t* __restrict__ tokens, int ctx, const float* __restrict__ tok,
                                                         const float* __restrict__ pos, const float* __restrict__ pre_g,
                                                         const float* __restrict__ pre_b, const float* __restrict__ g1,
                                                         const float* __restrict__ b1, int rows, int L, int W, int fmt,
                                                         uint16_t* __restrict__ a16, float* __restrict__ ones) {
  pdl_prologue();
  const int lane = threadIdx.x & 31, nwarps = (int)(gridDim.x * blockDim.x >> 5);
  for (int r = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); r < rows; r += nwarps) {  // warp-uniform
    const int s = r / L, l = r % L, nv = W >> 5;
    const float* src = tokens ? tok + (size_t)tokens[(size_t)s * ctx + l] * W : (l == 0 ? cls : x32 + (size_t)r * W);
    float v[kClipMaxWidth / 32], y[kClipMaxWidth / 32];
#pragma unroll
    for (int i = 0; i < kClipMaxWidth / 32; ++i)
      if (i < nv) v[i] = src[lane + 32 * i] + __ldg(pos + (size_t)l * W + lane + 32 * i);
    if (!tokens) {
      clip_ln(v, W, pre_g, pre_b, lane, y);
#pragma unroll
      for (int i = 0; i < kClipMaxWidth / 32; ++i)
        if (i < nv) v[i] = y[i];
    }
    clip_ln(v, W, g1, b1, lane, y);
    float* xr = x32 + (size_t)r * W;
    uint16_t* ar = a16 + (size_t)r * W;
#pragma unroll
    for (int i = 0; i < kClipMaxWidth / 32; ++i)
      if (i < nv) {
        xr[lane + 32 * i] = v[i];
        ar[lane + 32 * i] = cvt16(y[i], fmt);
      }
    if (lane == 0) ones[r] = 1.f;
  }
}

// Head LayerNorm, one warp per output row i < rows (warp-stride loop), over source row src(i) of x32:
//   tokens == null: src = i * stride (stride L: the class rows; 1: every row);
//   tokens: src = i * L + argmax_j tokens[i * ctx + j] (the first maximum, as torch.argmax returns it: the EOT position)
// out32 [rows, W] f32 and/or out16 [rows, W] 16-bit.
__global__ void __launch_bounds__(256) clip_head_ln_kernel(const float* __restrict__ x32, int rows, int stride, int L,
                                                           const int64_t* __restrict__ tokens, int ctx, const float* __restrict__ g,
                                                           const float* __restrict__ b, int W, int fmt, float* __restrict__ out32,
                                                           uint16_t* __restrict__ out16) {
  pdl_prologue();
  const int lane = threadIdx.x & 31, nwarps = (int)(gridDim.x * blockDim.x >> 5);
  for (int i = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); i < rows; i += nwarps) {  // warp-uniform
    size_t src = (size_t)i * stride;
    if (tokens) {
      long long best = LLONG_MIN;
      int arg = 0;
      for (int j = lane; j < ctx; j += 32) {
        const long long t = tokens[(size_t)i * ctx + j];
        if (t > best) {
          best = t;
          arg = j;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const long long ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        if (ob > best || (ob == best && oa < arg)) {
          best = ob;
          arg = oa;
        }
      }
      src = (size_t)i * L + arg;
    }
    const int nv = W >> 5;
    float v[kClipMaxWidth / 32], y[kClipMaxWidth / 32];
#pragma unroll
    for (int k = 0; k < kClipMaxWidth / 32; ++k)
      if (k < nv) v[k] = x32[src * W + lane + 32 * k];
    clip_ln(v, W, g, b, lane, y);
#pragma unroll
    for (int k = 0; k < kClipMaxWidth / 32; ++k)
      if (k < nv) {
        if (out32) out32[(size_t)i * W + lane + 32 * k] = y[k];
        if (out16) out16[(size_t)i * W + lane + 32 * k] = cvt16(y[k], fmt);
      }
  }
}

int clip_check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) set_error("%s launch failed: %s", what, cudaGetErrorString(e));
  return (int)e;
}

// Blocks of `threads` for n work items, capped at 65536: every kernel launched with it loops over its items with the grid's stride.
inline unsigned int grid_for(size_t n, int threads) {
  const size_t b = (n + threads - 1) / threads;
  return (unsigned int)(b < 65536 ? (b ? b : 1) : 65536);
}

int clip_sms() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 132;
}

// One K-major GEMM launch: C[M, N] = A[M, K] W[N, K]^T, epilogue set by `epi`.
template <typename Epi>
int clip_gemm(const uint16_t* A, int M, int K, const uint16_t* Wt, int N, int fmt, int sms, cudaStream_t st, Epi epi) {
  GemmGroup g;
  memset(&g, 0, sizeof(g));
  g.num = 1;
  g.fmt = fmt;
  const int bn = tile_for(sms, 16, MNK{M, N, K}).bn;
  if (setup_linear(g.p[0], A, M, K, K, Wt, N, K, bn)) return 1;
  epi(g.p[0]);
  return launch_gemm_group(g, bn, sms, st);
}

// The pre-norm blocks over the stream w.x32 (nseq sequences of L tokens); w.a16 holds ln_1 of block 0 on entry.  On return
// x32 is the transformer's output.
int clip_blocks(const uint8_t* pk, const ClipBlockPk* blk, int layers, const ClipWs& w, int nseq, int L, int W, int fmt, bool causal,
                int sms, cudaStream_t st) {
  auto F32 = [&](size_t off) { return reinterpret_cast<const float*>(pk + off); };
  auto W16 = [&](size_t off) { return reinterpret_cast<const uint16_t*>(pk + off); };
  const int M = nseq * L;
  int rc = 0;
  auto layernorm = [&](size_t gw, size_t gb) {
    LnArgs a;
    memset(&a, 0, sizeof(a));
    a.in = w.x32;
    a.ld_in = W;
    a.rows = M;
    a.d = W;
    a.gamma = F32(gw);
    a.beta = F32(gb);
    a.eps = 1e-5f;
    a.fmt = fmt;
    a.out16 = w.a16;
    a.ld16 = W;
    return launch_layernorm(a, st);
  };
  auto residual = [&](const float* bias) {
    return [=](GemmProblem& p) {
      p.bias = bias;
      p.resid = w.x32;
      p.ld_resid = W;
      p.out32 = w.x32;
      p.ld32 = W;
    };
  };
  for (int l = 0; l < layers; ++l) {
    const ClipBlockPk& b = blk[l];
    rc = clip_gemm(w.a16, M, W, W16(b.w_in), 3 * W, fmt, sms, st, [&](GemmProblem& p) {
      p.bias = F32(b.b_in);
      p.out16 = w.qkv16;
      p.ld16 = 3 * W;
    });
    if (rc) return rc;
    AttnArgs a;
    memset(&a, 0, sizeof(a));
    if (make_tmap_2d(&a.tm_qkv, w.qkv16, (uint64_t)M, (uint64_t)3 * W, (uint64_t)3 * W, 128, 64)) return 1;
    a.scale = 0.125f;  // 1 / sqrt(64)
    a.key_mask = w.ones;
    a.out = w.attn16;
    a.B = nseq;
    a.L = L;
    a.H = W / 64;
    a.dh = 64;
    a.d = W;
    a.fmt = fmt;
    a.causal = causal ? 1 : 0;
    rc = launch_attention(a, st);
    if (rc) return rc;
    rc = clip_gemm(w.attn16, M, W, W16(b.w_out), W, fmt, sms, st, residual(F32(b.b_out)));
    if (rc) return rc;
    rc = layernorm(b.ln2w, b.ln2b);
    if (rc) return rc;
    rc = clip_gemm(w.a16, M, W, W16(b.w_fc), 4 * W, fmt, sms, st, [&](GemmProblem& p) {
      p.bias = F32(b.b_fc);
      p.act = ACT_QUICKGELU;
      p.out16 = w.h16;
      p.ld16 = 4 * W;
    });
    if (rc) return rc;
    rc = clip_gemm(w.h16, M, 4 * W, W16(b.w_pr), W, fmt, sms, st, residual(F32(b.b_pr)));
    if (rc) return rc;
    if (l + 1 < layers) {
      rc = layernorm(blk[l + 1].ln1w, blk[l + 1].ln1b);
      if (rc) return rc;
    }
  }
  return 0;
}

}  // namespace

extern "C" {

int univtg_clip_num_params(const univtg_clip_config* cfg) {
  if (!clip_check_cfg(cfg, "univtg_clip_num_params")) return -1;
  return 8 + 12 * cfg->vision_layers + 5 + 12 * cfg->text_layers;
}

size_t univtg_clip_packed_bytes(const univtg_clip_config* cfg) {
  if (!clip_check_cfg(cfg, "univtg_clip_packed_bytes")) return 0;
  return clip_layout(*cfg).total;
}

int univtg_clip_pack_weights(const univtg_clip_config* cfg, const void* const* params, int32_t n_params, int32_t src_dtype, void* packed,
                             void* stream) {
  const char* fn = "univtg_clip_pack_weights";
  if (!clip_check_cfg(cfg, fn)) return 1;
  const int expect = univtg_clip_num_params(cfg);
  if (!params || n_params != expect) {
    set_error("%s: params must hold %d tensors, got %d", fn, expect, params ? n_params : 0);
    return 1;
  }
  if (src_dtype != 0 && src_dtype != 1) {
    set_error("%s: src_dtype %d must be 0 (f32) or 1 (fp16)", fn, src_dtype);
    return 1;
  }
  if (!packed) {
    set_error("%s: packed is null", fn);
    return 1;
  }
  for (int i = 0; i < n_params; ++i)
    if (!params[i]) {
      set_error("%s: params[%d] is null", fn, i);
      return 1;
    }
  const univtg_clip_config& c = *cfg;
  const ClipPacked L = clip_layout(c);
  const ClipShape s = clip_shape(c);
  const int fmt = c.operand_format;
  uint8_t* base = reinterpret_cast<uint8_t*>(packed);
  cudaStream_t st = (cudaStream_t)stream;
  int idx = 0;
  auto task = [&](size_t off, int kind, int rows, int cols, int ld) {
    const size_t n = kind == 0 ? (size_t)rows * ld : (size_t)rows * cols;
    launch_k(clip_pack_kernel, dim3(grid_for(n, 256)), dim3(256), 0, st, params[idx++], (int)src_dtype, (void*)(base + off), kind, rows,
             cols, ld, fmt);
  };
  auto blocks = [&](const ClipBlockPk* blk, int layers, int W) {
    for (int l = 0; l < layers; ++l) {
      const ClipBlockPk& b = blk[l];
      task(b.w_in, 0, 3 * W, W, W);
      task(b.b_in, 1, 1, 3 * W, 0);
      task(b.w_out, 0, W, W, W);
      task(b.b_out, 1, 1, W, 0);
      task(b.ln1w, 1, 1, W, 0);
      task(b.ln1b, 1, 1, W, 0);
      task(b.w_fc, 0, 4 * W, W, W);
      task(b.b_fc, 1, 1, 4 * W, 0);
      task(b.w_pr, 0, W, 4 * W, 4 * W);
      task(b.b_pr, 1, 1, W, 0);
      task(b.ln2w, 1, 1, W, 0);
      task(b.ln2b, 1, 1, W, 0);
    }
  };
  const int Wv = c.vision_width, Wt = c.text_width, E = c.embed_dim;
  task(L.conv16, 0, Wv, 3 * c.patch_size * c.patch_size, s.kpad);
  task(L.cls, 1, 1, Wv, 0);
  task(L.vpos, 1, s.lp, Wv, 0);
  task(L.ln_pre_w, 1, 1, Wv, 0);
  task(L.ln_pre_b, 1, 1, Wv, 0);
  blocks(L.vblk, c.vision_layers, Wv);
  task(L.ln_post_w, 1, 1, Wv, 0);
  task(L.ln_post_b, 1, 1, Wv, 0);
  task(L.vproj16, 2, Wv, E, 0);  // visual.proj [Wv, E] -> [E, Wv]
  task(L.tok, 1, c.vocab_size, Wt, 0);
  task(L.tpos, 1, c.context_length, Wt, 0);
  blocks(L.tblk, c.text_layers, Wt);
  task(L.ln_f_w, 1, 1, Wt, 0);
  task(L.ln_f_b, 1, 1, Wt, 0);
  task(L.tproj16, 2, Wt, E, 0);  // text_projection [Wt, E] -> [E, Wt]
  return clip_check_launch(fn);
}

size_t univtg_clip_workspace_bytes(const univtg_clip_config* cfg, int32_t n_images, int32_t n_texts, int32_t text_len) {
  if (!clip_check_cfg(cfg, "univtg_clip_workspace_bytes")) return 0;
  if (n_images < 0 || n_texts < 0 || text_len < 0 || text_len > cfg->context_length) {
    set_error("univtg_clip_workspace_bytes: n_images %d, n_texts %d must be >= 0 and text_len %d in [0, context_length %d]", n_images,
              n_texts, text_len, cfg->context_length);
    return 0;
  }
  const size_t a = clip_vision_ws_bytes(*cfg, (size_t)n_images), b = clip_text_ws_bytes(*cfg, (size_t)n_texts, (size_t)text_len);
  return a > b ? a : b;
}

int univtg_clip_num_launches(const univtg_clip_config* cfg, int32_t tower, int32_t text_outputs) {
  if (!clip_check_cfg(cfg, "univtg_clip_num_launches")) return -1;
  if (tower == 0) return 3 + (7 * cfg->vision_layers - 1) + 2;
  if (tower == 1) return 1 + (7 * cfg->text_layers - 1) + ((text_outputs & 1) ? 1 : 0) + ((text_outputs & 2) ? 2 : 0);
  set_error("univtg_clip_num_launches: tower %d must be 0 (image) or 1 (text)", tower);
  return -1;
}

int univtg_clip_encode_image(const univtg_clip_config* cfg, const void* packed, const void* pixels, int32_t pixel_kind, int32_t n,
                             void* ws, size_t ws_bytes, float* out, void* stream) {
  const char* fn = "univtg_clip_encode_image";
  if (!clip_check_cfg(cfg, fn)) return 1;
  const univtg_clip_config& c = *cfg;
#define CLIP_ARG(cond, ...)  \
  if (!(cond)) {             \
    set_error(__VA_ARGS__);  \
    return 1;                \
  }
  CLIP_ARG(packed, "%s: packed is null", fn);
  CLIP_ARG(pixels, "%s: pixels is null", fn);
  CLIP_ARG(pixel_kind == 0 || pixel_kind == 1, "%s: pixel_kind %d must be 0 (uint8 [n, R, R, 3]) or 1 (f32 [n, 3, R, R])", fn, pixel_kind);
  CLIP_ARG(n >= 1 && n <= 65535, "%s: n %d must be in [1, 65535] (one attention grid z-slice per sequence)", fn, n);
  CLIP_ARG(out, "%s: out is null", fn);
  CLIP_ARG(ws, "%s: ws is null", fn);
  const size_t need = clip_vision_ws_bytes(c, (size_t)n);
  CLIP_ARG(ws_bytes >= need, "%s: ws_bytes %zu < %zu needed for %d frames", fn, ws_bytes, need, n);
  const ClipPacked P = clip_layout(c);
  const ClipShape s = clip_shape(c);
  const int W = c.vision_width, fmt = c.operand_format, M = n * s.lp, sms = clip_sms();
  const uint8_t* pk = reinterpret_cast<const uint8_t*>(packed);
  auto F32 = [&](size_t off) { return reinterpret_cast<const float*>(pk + off); };
  auto W16 = [&](size_t off) { return reinterpret_cast<const uint16_t*>(pk + off); };
  const ClipWs w = clip_ws((size_t)M, W, n, (size_t)n * s.pc * s.kpad, reinterpret_cast<uint8_t*>(ws));
  cudaStream_t st = (cudaStream_t)stream;

  launch_k(clip_frames_kernel, dim3(grid_for((size_t)n * s.pc * s.kpad, 256)), dim3(256), 0, st, pixels, (int)pixel_kind, (int)n,
           c.image_resolution, c.patch_size, s.grid, s.kpad, fmt, w.patch16);
  int rc = clip_check_launch("clip_frames");
  if (rc) return rc;
  // conv1 as a GEMM: patch rows t * pc + p land on stream rows t * lp + 1 + p (row 0 of each frame is the class token)
  rc = clip_gemm(w.patch16, n * s.pc, s.kpad, W16(P.conv16), W, fmt, sms, st, [&](GemmProblem& p) {
    p.rps_in = s.pc;
    p.rps_out = s.lp;
    p.row_off = 1;
    p.out32 = w.x32;
    p.ld32 = W;
  });
  if (rc) return rc;
  launch_k(clip_embed_kernel, dim3(grid_for((size_t)M * 32, 256)), dim3(256), 0, st, w.x32, F32(P.cls), (const int64_t*)nullptr, 0,
           (const float*)nullptr, F32(P.vpos), F32(P.ln_pre_w), F32(P.ln_pre_b), F32(P.vblk[0].ln1w), F32(P.vblk[0].ln1b), M, s.lp, W,
           fmt, w.a16, w.ones);
  rc = clip_check_launch("clip_embed");
  if (rc) return rc;
  rc = clip_blocks(pk, P.vblk, c.vision_layers, w, n, s.lp, W, fmt, false, sms, st);
  if (rc) return rc;
  launch_k(clip_head_ln_kernel, dim3(grid_for((size_t)n * 32, 256)), dim3(256), 0, st, (const float*)w.x32, (int)n, s.lp, s.lp,
           (const int64_t*)nullptr, 0, F32(P.ln_post_w), F32(P.ln_post_b), W, fmt, (float*)nullptr, w.head16);
  rc = clip_check_launch("clip_head_ln");
  if (rc) return rc;
  return clip_gemm(w.head16, n, W, W16(P.vproj16), c.embed_dim, fmt, sms, st, [&](GemmProblem& p) {
    p.out32 = out;
    p.ld32 = c.embed_dim;
  });
}

int univtg_clip_encode_text(const univtg_clip_config* cfg, const void* packed, const int64_t* tokens, int32_t n, int32_t ctx_used,
                            void* ws, size_t ws_bytes, float* last_hidden, float* pooled, void* stream) {
  const char* fn = "univtg_clip_encode_text";
  if (!clip_check_cfg(cfg, fn)) return 1;
  const univtg_clip_config& c = *cfg;
  CLIP_ARG(packed, "%s: packed is null", fn);
  CLIP_ARG(tokens, "%s: tokens is null", fn);
  CLIP_ARG(n >= 1 && n <= 65535, "%s: n %d must be in [1, 65535] (one attention grid z-slice per sequence)", fn, n);
  CLIP_ARG(ctx_used >= 1 && ctx_used <= c.context_length, "%s: ctx_used %d must be in [1, context_length %d]", fn, ctx_used,
           c.context_length);
  CLIP_ARG(last_hidden || pooled, "%s: last_hidden and pooled are both null", fn);
  CLIP_ARG(ws, "%s: ws is null", fn);
  const size_t need = clip_text_ws_bytes(c, (size_t)n, (size_t)ctx_used);
  CLIP_ARG(ws_bytes >= need, "%s: ws_bytes %zu < %zu needed for %d texts of %d positions", fn, ws_bytes, need, n, ctx_used);
  cudaStream_t st = (cudaStream_t)stream;
  const int C = c.context_length;
  {  // the ids index token_embedding and pick the pooled row: check them before any kernel reads them
    std::vector<int64_t> h((size_t)n * C);
    cudaError_t e = cudaMemcpyAsync(h.data(), tokens, h.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
      set_error("%s: reading tokens back failed: %s", fn, cudaGetErrorString(e));
      return (int)e;
    }
    for (int i = 0; i < n; ++i) {
      int arg = 0;
      for (int j = 0; j < C; ++j) {
        const int64_t t = h[(size_t)i * C + j];
        CLIP_ARG(t >= 0 && t < c.vocab_size, "%s: tokens[%d, %d] = %lld is outside [0, vocab_size %d)", fn, i, j, (long long)t,
                 c.vocab_size);
        if (t > h[(size_t)i * C + arg]) arg = j;
      }
      CLIP_ARG(!pooled || arg < ctx_used, "%s: tokens row %d has its argmax (EOT) at position %d >= ctx_used %d", fn, i, arg, ctx_used);
    }
  }
#undef CLIP_ARG
  const ClipPacked P = clip_layout(c);
  const int W = c.text_width, fmt = c.operand_format, Lc = ctx_used, M = n * Lc, sms = clip_sms();
  const uint8_t* pk = reinterpret_cast<const uint8_t*>(packed);
  auto F32 = [&](size_t off) { return reinterpret_cast<const float*>(pk + off); };
  auto W16 = [&](size_t off) { return reinterpret_cast<const uint16_t*>(pk + off); };
  const ClipWs w = clip_ws((size_t)M, W, n, 0, reinterpret_cast<uint8_t*>(ws));

  launch_k(clip_embed_kernel, dim3(grid_for((size_t)M * 32, 256)), dim3(256), 0, st, w.x32, (const float*)nullptr, tokens, C, F32(P.tok),
           F32(P.tpos), (const float*)nullptr, (const float*)nullptr, F32(P.tblk[0].ln1w), F32(P.tblk[0].ln1b), M, Lc, W, fmt, w.a16,
           w.ones);
  int rc = clip_check_launch("clip_embed");
  if (rc) return rc;
  rc = clip_blocks(pk, P.tblk, c.text_layers, w, n, Lc, W, fmt, true, sms, st);
  if (rc) return rc;
  if (last_hidden) {
    launch_k(clip_head_ln_kernel, dim3(grid_for((size_t)M * 32, 256)), dim3(256), 0, st, (const float*)w.x32, M, 1, Lc,
             (const int64_t*)nullptr, 0, F32(P.ln_f_w), F32(P.ln_f_b), W, fmt, last_hidden, (uint16_t*)nullptr);
    rc = clip_check_launch("clip_head_ln");
    if (rc) return rc;
  }
  if (pooled) {
    launch_k(clip_head_ln_kernel, dim3(grid_for((size_t)n * 32, 256)), dim3(256), 0, st, (const float*)w.x32, (int)n, 0, Lc, tokens, C,
             F32(P.ln_f_w), F32(P.ln_f_b), W, fmt, (float*)nullptr, w.head16);
    rc = clip_check_launch("clip_head_ln");
    if (rc) return rc;
    rc = clip_gemm(w.head16, n, W, W16(P.tproj16), c.embed_dim, fmt, sms, st, [&](GemmProblem& p) {
      p.out32 = pooled;
      p.ld32 = c.embed_dim;
    });
  }
  return rc;
}

}  // extern "C"
