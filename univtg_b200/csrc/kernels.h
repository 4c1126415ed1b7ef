// Internal (C++) interface between the C-ABI layer (api.cu) and the kernel translation units.
#pragma once
#include <string.h>
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace uv {

constexpr int GEMM_BM = 128;  // tile rows: two consumer warpgroups of wgmma M = 64
constexpr int GEMM_BK = 64;   // one 128-byte swizzle span of 16-bit elements
constexpr int GEMM_MAX_GROUP = 4;

enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_QUICKGELU = 3 };  // QuickGELU: x * sigmoid(1.702 x) (CLIP MLP)

// TMA coordinate rule of one operand for the k-block (tap, kk) of the output tile whose first
// row (A) / first column (B) is `mn0`:
//   c0 = base0 + mn0*mn0s + tap*tap0 + kk*64*k0s      (innermost / contiguous coordinate)
//   c1 = base1 + mn0*mn1s + tap*tap1 + kk*64*k1s      (row coordinate)
struct OperandCoord {
  int base0, mn0s, tap0, k0s;
  int base1, mn1s, tap1, k1s;
};

// One C[M,N] = epilogue(A[M,K] * B[N,K]^T) problem.  Up to GEMM_MAX_GROUP problems share one
// persistent launch (tiles of all problems are interleaved over the SMs).
struct GemmProblem {
  // 16-bit operand maps, 128-byte swizzle.
  //   K-major  operand (contraction contiguous): dims {K, rows},  box {64, 128 (A) | BN (B)}
  //   MN-major operand (contraction is the row): dims {MN, Krows}, box {64, 64}, one box per 64 M/N elements
  CUtensorMap tm_a;
  CUtensorMap tm_b;
  OperandCoord ca, cb;
  int a_mn, b_mn;    // 1: operand is MN-major in memory
  int b_box_rows;    // rows of tm_b's TMA box (K-major B): must equal the launch's bn (bn/2 for cluster pairs); checked at launch
  int M, N;
  int taps;          // 1 = plain; 3 = k=3 conv expressed as 3 K segments
                     // Forward conv (conv_fwd_problem, plan.h) over the conv-head layout [B*(Lv+1)+2, C] (buffer row = logical row + 1):
                     // A rows 0 and M+1 and every sample's separator row must hold zeros; with rps_in = rps_out = Lv+1, row_off = 1 and
                     // zero_sep the epilogue writes buffer rows 1..M (separators as exact zeros) and never rows 0 and M+1.
  int kblk_per_tap;  // 64-wide k-blocks per tap
  int ksplit;        // >=1; k-blocks are split over `ksplit` tiles that accumulate atomically into out32, which the caller must have
                     // zeroed (or filled with what the sum should be added to).  ksplit > 1 and `accumulate` are rejected together
                     // with act, resid, out16, out16p, out32_id or dact16, which are not additive over partial sums.
  // ---- epilogue:  v = act(acc + bias[n]) * alpha * row_scale[b(m)]  (+ resid[orow, n]) ----
  const float* bias;
  float alpha;
  int act;
  const float* row_scale;  // [num samples] or null
  int rps_in;              // rows per sample in the M index space (0: single sample)
  int rps_out;             // out row = (m / rps_in) * rps_out + (m % rps_in) + row_off
  int row_off;
  int zero_sep;            // rows with (m % rps_in) == rps_in-1 are stored as exact zeros (conv separator rows)
  const float* resid;      // fp32, indexed by out row
  int ld_resid;
  const float* addtab;     // fp32 table indexed by m (sine position table); only used for out16p
  int ld_addtab;
  float* out32;            // fp32 at remapped rows
  int ld32;
  float* out32_id;         // fp32 at identity rows (m)
  int ld32_id;
  uint16_t* out16;         // 16-bit at remapped rows
  uint16_t* out16p;        // 16-bit(v + addtab[m, n]) at remapped rows (same leading dim as out16)
  int ld16;
  int accumulate;          // out32 += v (atomic) instead of out32 = v
  // ---- backward-pass extras (all optional) ----
  int a_fmt, b_fmt;        // per-operand 16-bit format override (-1: group fmt); gradients travel as bf16, activations as fp16
  int out_fmt;             // format of out16 / out16p (-1: group fmt)
  const float* aux32;      // fp32 matrix indexed like out32 (remapped rows)
  int ld_aux;
  int aux_mode;            // 1: v *= gelu'(aux)   2: v *= aux (e.g. a dropout mask incl. its 1/(1-p) scale)
  const uint16_t* mask16;  // 16-bit activation indexed like out16: v = 0 where mask16 <= 0 (ReLU backward)
  int ld_mask;
  float* pre32;            // fp32 (acc + bias) BEFORE the activation, indexed like out32
  int ld_pre;
  uint16_t* dact16;        // 16-bit d act / d pre-activation at (acc + bias), indexed like out16 (ACT_GELU: saved for the backward, which
  int ld_dact;             //   then multiplies by it - mask16 + mask_mul - instead of re-evaluating erf / exp on an fp32 copy)
  int mask_mul;            // 1: v *= mask16 (an activation derivative) instead of zeroing where mask16 <= 0
  float colsum_scale;      // factor applied to the column sums (1/loss-scale for bias gradients)
  float* colsum;           // fp32 [N]: atomically accumulates the column sums of the stored values (bias gradients)
  int cs32;                // column stride of out32 (0/1: dense); 3 writes a Conv1d weight-gradient tap in [n, c, 3] layout
  int skip_sep;            // rows with (m % rps_in) == rps_in-1 are not stored at all
  int b_3d;                // MN-major B through ONE 3-D TMA box per k-block: number of 64-wide N blocks in the box (0: one 2-D box per block)
  int vec_ok;              // set by launch_gemm_group: 1 = every pointer / leading dimension allows 128-bit accesses, 2 = 256-bit
};

struct GemmGroup {
  int num;
  int fmt;  // 0 fp16, 1 bf16
  int bn;   // tile width of this launch (set by launch_gemm_group)
  int cluster;  // 2: CTA pairs share the B tile through TMA multicast (K-major B maps must then use box rows = bn/2)
  int split;    // 1: fp16x3 (fmt 0, cluster 1, K-major operands): tm_a / tm_b are make_tmap_split pairs, every product is
                //    A_hi B_hi + A_lo B_hi + A_hi B_lo, and out16 / out16p are stored as hi / lo pairs
  long long lo16;  // split: elements from out16 / out16p to their lo planes
  unsigned long long* dbg;  // optional [gridDim.x][8] %globaltimer stamps per CTA (profiling aid), normally null
  GemmProblem p[GEMM_MAX_GROUP];
};

// ---- static deal of a launch's work units over its persistent CTAs ----
// A unit is one output tile (CL = 2: tile pair) of one k-split of one problem.  Units are numbered longest first: problems in
// deal order (k-blocks per unit descending, ties in problem order; launch_gemm_group launches the problems so ordered), a
// problem's units in tile order.  They are dealt in waves of one unit per CTA whose direction alternates (a snake): the CTA
// that draws the longest unit of one wave draws the shortest of the next.  Round r of CTA c (of n) runs unit gemm_deal_unit(n, c, r); every unit is run exactly once.
__host__ __device__ __forceinline__ int gemm_deal_unit(int n, int c, int r) { return r * n + ((r & 1) ? n - 1 - c : c); }
// k-blocks of one unit of problem `pr` (its last split may be shorter); split: fp16x3 walks every k-block three times.
__host__ __device__ __forceinline__ int gemm_unit_kblocks(const GemmProblem& pr, bool split) {
  const int total_kb = pr.taps * pr.kblk_per_tap * (split ? 3 : 1);
  return (total_kb + pr.ksplit - 1) / pr.ksplit;
}
// Puts g's problems in deal order; perm (optional) receives the original index of each.
void gemm_deal_order(GemmGroup& g, int* perm);

// bn: tile width, multiple of 16 in [32, 256] (multiple of 64 when a problem has an MN-major B).  A and B of a problem must share
// one 16-bit format.  Returns cudaError_t as int.  used_full (optional): 1 when the FULL epilogue variant was launched, 0 for the lean one.
int launch_gemm_group(GemmGroup& g, int bn, int num_sms, cudaStream_t stream, int* used_full = nullptr);
// Tile width and per-problem split-K factors that minimise the modelled time of problems sharing one launch (step 16: K-major B,
// 64: MN-major B).  max_split[p] (a power of two): split limit of problem p, 1 for a problem whose epilogue cannot accumulate.
struct TileChoice {
  int bn;
  int ksplit;                  // the largest of ks
  int ks[GEMM_MAX_GROUP];      // split-K factor of each problem
};
TileChoice choose_tile(const int* Ms, const int* Ns, const int* kblocks, const int* max_split, int num, int num_sms, int step);
// The deal of gemm_wgmma_kernel (CL = 1) for problems M x N with kblocks k-blocks split ksplit ways at width bn: cta[u] receives the
// CTA that runs unit u (units problem by problem, in each problem's tile order; -1 if no CTA runs it, -2 if two do).  Returns the
// number of units (also when it exceeds cap, in which case nothing past cap is written), or -1 for bad arguments.
int gemm_deal_ctas(const int* Ms, const int* Ns, const int* kblocks, const int* ksplit, int num, int num_sms, int bn, int* cta, int cap);
// MN-major B operand [rows = K, cols = N] (N contiguous): a 3-D view {64, K, N/64} lets one TMA instruction fetch the whole
// 64 x bn tile of a k-block (fewer TMA operations per k-block than one 2-D box per 64-wide block); needs cols % 64 == 0.
int make_tmap_b_mn(GemmProblem& p, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, int bn);

// Encode a 2-D tensor map over a row-major 16-bit matrix [rows, cols] with row pitch `ld` elements,
// box {box_cols, box_rows}, 128-byte swizzle, zero fill out of bounds.  Returns 0 on success.
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                 uint32_t box_cols);

// fp16x3 pair: a 3-D map {cols, rows, 2} over a hi plane and the lo plane `lo_elems` elements after it (same rows, cols, pitch).
int make_tmap_split(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld_elems, uint32_t box_rows,
                    uint32_t box_cols, uint64_t lo_elems);

void set_gemm_timeline_buffer(unsigned long long* buf);  // debugging: stamps for every following GEMM launch
const char* last_error();
void set_error(const char* fmt, ...);
// ---- kernel launches with programmatic dependent launch (PDL) ----
// Every kernel of this library starts with pdl_prologue() (griddepcontrol.launch_dependents + griddepcontrol.wait, ptx.cuh):
// the next kernel in the stream may be scheduled while this one is still running and blocks at its own
// griddepcontrol.wait until this grid has completed and flushed - the launch latency and the next kernel's prologue
// (barrier init, tensor-map prefetch) disappear under the current kernel's tail.  UNIVTG_PDL=0 disables it.
bool pdl_enabled();
long long* launch_counter();  // kernels launched by this library since it was loaded (bench accounting: gpu_launches)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  ++*launch_counter();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// 16-bit operand copies written by the fused AdamW step itself (optim.cu): the big GEMM weight matrices, described as ranges of the
// flat parameter buffer.  kind 0: [rows, cols] -> 16-bit [rows, ld] (K padding beyond cols stays zero); kind 1: Conv1d weight
// [N = rows, C = cols, 3] -> 16-bit [N, 3C] with w2[n, t*C + c] = w[n, c, t].
struct PackSeg {
  long long start4, end4;  // float4 index range inside the flat buffer
  void* dst;
  int kind, rows, cols, ld;
};
constexpr int kMaxPackSegs = 40;
struct PackSegTable {
  int n, fmt;
  PackSeg s[kMaxPackSegs];
};

// device-resident optimizer state of univtg_adamw_step_dev (null: lr / step by value)
struct AdamDevState {
  const float* lr;         // device fp32 scalar
  int32_t* step;           // device int32: completed updates; advanced by the kernel when the step is not skipped
  const float* bc_table;   // device fp32 [table_len][2]: (bc1, bc2_sqrt) of steps 1 .. table_len (adamw_bias_row)
  int32_t table_len;
};
void adamw_bias_row(float beta1, float beta2, int32_t step, float* bc1, float* bc2_sqrt);
int adamw_step_impl(float* params, float* grads, float* exp_avg, float* exp_avg_sq, size_t n, float lr, float beta1, float beta2,
                    float eps, float weight_decay, int32_t step, float max_grad_norm, int32_t write_clipped_grads, float* scratch3,
                    const PackSegTable* segs, void* stream, const AdamDevState* dev = nullptr);


}  // namespace uv
