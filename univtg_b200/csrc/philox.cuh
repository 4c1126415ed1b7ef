// Counter-based random numbers for the train-mode randomness of the path, generated INSIDE the kernels that consume it
// (no mask tensors in HBM, regenerated bit-identically by the backward):
//   * input dropout   nn.Dropout(p) of every LinearLayer (reference model/univtg.py:394,401): multiplier 0 or 1/(1-p) per element
//   * DropPath        floor(keep + U[0,1)) / keep per sample and residual branch (model/transformer_encoder_droppath.py:154-167)
//   * attention dropout  F.dropout of the softmax probabilities in every encoder layer's nn.MultiheadAttention (args.dropout):
//                     multiplier 0 or 1/(1-p) per (layer, b, h, query, key), applied inside the attention kernels
// Philox4x32-10 (Salmon et al., SC'11; the generator family torch's CUDA RNG uses), keyed by (seed, stream), counter = (row,
// column / 8); one call yields eight 16-bit lanes = the dropout decisions of eight consecutive columns of a row.  The draws are NOT torch's draws for the same seed
// (torch's element-to-counter mapping depends on its launch geometry); parity tests read the multipliers back through
// univtg_dropout_mask / univtg_droppath_scales and hand them to the oracle, and model.reference_rng_order = True keeps the
// torch-drawn path for bit-parity with the reference's RNG stream.
#pragma once
#include <stdint.h>

namespace uv {

struct DropSpec {
  unsigned long long seed;
  const unsigned long long* seed_ptr;  // non-null: the seed lives in device memory (read once per kernel, see drop_resolve)
  unsigned int stream;  // which mask of the step (projector layer / modality)
  unsigned int thresh;  // element kept iff its 16-bit lane >= thresh (thresh = round(p * 65536))
  float scale;          // 1 / (1 - p)
  int on;               // 0: no dropout
};

// A captured CUDA graph replays its kernels with the arguments of the capture, so a seed passed by value would draw the same
// masks on every replay.  With seed_ptr set the seed is read from device memory instead (written ahead of the step by
// univtg_rng_advance): once per kernel, after the PDL wait, never inside the Philox loops.
__device__ __forceinline__ unsigned long long drop_seed(const DropSpec& s) { return s.seed_ptr != nullptr ? *s.seed_ptr : s.seed; }
__device__ __forceinline__ DropSpec drop_resolve(const DropSpec& s) {
  DropSpec r = s;
  if (s.on) r.seed = drop_seed(s);
  return r;
}
__device__ __forceinline__ DropSpec drop_with_seed(const DropSpec& s, unsigned long long seed) {
  DropSpec r = s;
  r.seed = seed;
  return r;
}
__device__ __forceinline__ unsigned long long dp_seed_of(unsigned long long seed, const unsigned long long* seed_ptr) {
  return seed_ptr != nullptr ? *seed_ptr : seed;
}

__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned int hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const unsigned int hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}

// One Philox call = the decisions of the eight consecutive columns [8 cb, 8 cb + 8) of row `row` (row-aligned blocks: threads that
// own neighbouring columns of a row share a call whatever the row length is).
__device__ __forceinline__ uint4 drop_block(const DropSpec& s, unsigned int row, unsigned int cb) {
  return philox4x32_10(make_uint4(cb, row, s.stream, 0x756e6976u), make_uint2((unsigned int)s.seed, (unsigned int)(s.seed >> 32)));
}
__device__ __forceinline__ unsigned int drop_lane(const uint4& r, unsigned int lane) {  // lane in [0, 8)
  const unsigned int w = lane < 4 ? (lane < 2 ? r.x : r.y) : (lane < 6 ? r.z : r.w);
  return (lane & 1) ? (w >> 16) : (w & 0xffffu);
}
__device__ __forceinline__ float drop_pick(const DropSpec& s, const uint4& r, unsigned int lane) {
  return drop_lane(r, lane) >= s.thresh ? s.scale : 0.f;
}
// multiplier of element (row, col)
__device__ __forceinline__ float drop_mul1(const DropSpec& s, unsigned int row, unsigned int col) {
  const uint4 r = drop_block(s, row, col >> 3);
  return drop_pick(s, r, col & 7);
}
// multipliers of columns col .. col+3 of `row`, col % 4 == 0 (one Philox call)
__device__ __forceinline__ float4 drop_mul4(const DropSpec& s, unsigned int row, unsigned int col) {
  const uint4 r = drop_block(s, row, col >> 3);
  const unsigned int w0 = (col & 4) ? r.z : r.x, w1 = (col & 4) ? r.w : r.y;
  float4 m;
  m.x = (w0 & 0xffffu) >= s.thresh ? s.scale : 0.f;
  m.y = (w0 >> 16) >= s.thresh ? s.scale : 0.f;
  m.z = (w1 & 0xffffu) >= s.thresh ? s.scale : 0.f;
  m.w = (w1 >> 16) >= s.thresh ? s.scale : 0.f;
  return m;
}
// all eight multipliers of block cb of `row`
__device__ __forceinline__ void drop_mul8(const DropSpec& s, unsigned int row, unsigned int cb, float (&m)[8]) {
  const uint4 r = drop_block(s, row, cb);
  const unsigned int w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    m[2 * k] = (w[k] & 0xffffu) >= s.thresh ? s.scale : 0.f;
    m[2 * k + 1] = (w[k] >> 16) >= s.thresh ? s.scale : 0.f;
  }
}
// DropPath scale of (site, sample): u = 24-bit uniform in [0, 1) like torch.rand; floor(keep + u) / keep
__device__ __forceinline__ float droppath_scale(unsigned long long seed, unsigned int index, float keep) {
  const uint4 r = philox4x32_10(make_uint4(index, 0u, 0x64726f70u, 0x70617468u), make_uint2((unsigned int)seed, (unsigned int)(seed >> 32)));
  const float u = (float)(r.x >> 8) * (1.0f / 16777216.0f);
  return floorf(keep + u) / keep;
}

// ---- attention-probability dropout (F.dropout(attn, p) inside nn.MultiheadAttention, transformer_encoder_droppath.py:93) ----
// One multiplier per (layer = s.stream, bh = b * H + h, query i, key j), same thresh / scale as input dropout.  One Philox call
// covers query rows {i0, i0 + 8} x keys {j0, j0 + 1, j0 + 8, j0 + 9}, i0 = i with bit 3 cleared, j0 = j with bits 0 and 3
// cleared; its word 2 * (bit 3 of i) + (bit 3 of j) holds key bit 0 = 0 in the low and = 1 in the high 16-bit lane.  That block
// is exactly what one thread of the forward wgmma kernel holds for two adjacent 8-key accumulator blocks (one call per 8
// elements); the key-major backward uses 4 of the 8 lanes of each call; the SIMT kernels and the materialiser make one call per
// element.  The constant counter word 0x61740000 + layer keeps these streams apart from input dropout (0x756e6976) and DropPath.
__device__ __forceinline__ uint4 attn_drop_block(const DropSpec& s, unsigned int bh, unsigned int i0, unsigned int j0) {
  return philox4x32_10(make_uint4(j0, i0, bh, 0x61740000u + s.stream), make_uint2((unsigned int)s.seed, (unsigned int)(s.seed >> 32)));
}
// 16-bit lane of (i, j) in the call attn_drop_block(s, bh, i & ~8, j & ~9)
__device__ __forceinline__ unsigned int attn_drop_lane(const uint4& r, unsigned int i, unsigned int j) {
  return drop_lane(r, 4u * ((i >> 3) & 1u) + 2u * ((j >> 3) & 1u) + (j & 1u));
}
__device__ __forceinline__ float attn_drop_mul1(const DropSpec& s, unsigned int bh, unsigned int i, unsigned int j) {
  const uint4 r = attn_drop_block(s, bh, i & ~8u, j & ~9u);
  return attn_drop_lane(r, i, j) >= s.thresh ? s.scale : 0.f;
}

// Seed sequence of univtg_rng_advance / univtg_rng_seed_at: the k-th output of splitmix64 (Steele et al., OOPSLA'14) started at
// `base`, so consecutive replays get well-separated Philox keys.
__host__ __device__ __forceinline__ unsigned long long rng_seed_at(unsigned long long base, unsigned long long k) {
  unsigned long long z = base + k * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

inline DropSpec make_drop_spec(unsigned long long seed, unsigned int stream, float p) {
  DropSpec s;
  s.seed = seed;
  s.seed_ptr = nullptr;
  s.stream = stream;
  s.on = p > 0.f ? 1 : 0;
  const float pc = p < 0.f ? 0.f : (p > 0.999f ? 0.999f : p);
  s.thresh = (unsigned int)(pc * 65536.0f + 0.5f);
  s.scale = 1.0f / (1.0f - pc);
  return s;
}

}  // namespace uv
