// Shared helpers for libpgnn_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/pgnn_b200.h"

#include <atomic>
#include <utility>
extern thread_local int g_pgnn_last_cuda_error;
extern std::atomic<long long> g_pgnn_kernel_launches;  // every kernel this library enqueues (pgnn_kernel_launch_count)
// Per-kernel timing mode (pgnn_profile_enable): every launch is bracketed by a CUDA event pair on its own stream, so that
// a caller can read each kernel's duration inside the real step (warm L2, true operand residency) without a profiler.
extern std::atomic<int> g_pgnn_profile_on;
void pgnn_profile_mark(const void* kernel, cudaStream_t st, bool after);

// Device error word of the current device (lazily allocated, zeroed): kernels that consume indices OR a PGNN_DEVERR_* bit into
// it instead of reading or writing out of range; pgnn_device_error_flags() reads it back.  May return null (then unchecked).
unsigned int* pgnn_error_flag_ptr();

#define PGNN_CHECK_ARG(cond)            \
  do {                                  \
    if (!(cond)) return PGNN_EINVAL;    \
  } while (0)

#define PGNN_CUDA(call)                       \
  do {                                        \
    cudaError_t e__ = (call);                 \
    if (e__ != cudaSuccess) {                 \
      g_pgnn_last_cuda_error = (int)e__;      \
      return PGNN_ECUDA;                      \
    }                                         \
  } while (0)

#define PGNN_LAUNCH_CHECK()                                        \
  do {                                                             \
    g_pgnn_kernel_launches.fetch_add(1, std::memory_order_relaxed); \
    PGNN_CUDA(cudaGetLastError());                                 \
  } while (0)

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t align_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// Optional column reductions fused into the tensor-core GEMM epilogue (the output tile is already staged in shared
// memory there).  All outputs must be zeroed by the caller; every CTA adds its tile's contribution with atomics.
constexpr int kMaxHookQ = 16;  // columns of S the epilogue holds per row (its shared-memory slice is [128][kMaxHookQ])
struct PgnnGemmHooks {
  float* colsum = nullptr;   // [N]     += sum over rows of the (final) output              -> bias gradients
  double* stats = nullptr;   // [2][N]  += sum, sum of squares (fp64)                        -> BatchNorm batch statistics
  const float* S = nullptr;  // [M][Q]  per-row weights: gT[q][n] += sum_m S[m][q] out[m][n] -> bond-table gradients
  int Q = 0;                 // 1 <= Q <= kMaxHookQ when S is set
  float* gT = nullptr;       // rows [0, q_split)
  float* gT2 = nullptr;      // rows [q_split, Q)
  int q_split = 0;
  int64_t ldt = 0;
  bool any() const { return colsum || stats || S; }
};

// BatchNorm finalisation folded into the consumer kernel: from the fp64 column sums `acc` ([2][C]: sum, sum of squares
// over M rows) every CTA derives scale/shift itself; CTA 0 also performs the module-state updates of torch.nn.BatchNorm1d.
struct PgnnBnFold {
  const double* acc = nullptr;
  const float* gamma = nullptr;
  const float* beta = nullptr;
  float* running_mean = nullptr;
  float* running_var = nullptr;
  int64_t* nbt = nullptr;
  float* save_mean = nullptr;
  float* save_invstd = nullptr;
  float momentum = 0.1f, eps = 1e-5f;
  int M = 0;
  double inv_m = 0.0, unbias = 1.0;  // 1 / M and M / (M - 1), formed on the host (set_rows)
  void set_rows(int rows) {
    M = rows;
    inv_m = rows > 0 ? 1.0 / (double)rows : 0.0;
    unbias = rows > 1 ? (double)rows / (double)(rows - 1) : 1.0;
  }
};

// The BatchNorm pre-activation, defined once: y = act(fmaf(x, scale, shift)) with scale = gamma * invstd and
// shift = fmaf(-mean, scale, beta), all in fp32 with one rounding each.  Every forward apply (norm.cu, and the gathers of
// aggregate.cu that apply the previous layer's BatchNorm + ReLU on load) computes this expression, and every backward sweep
// recomputes it bit for bit from save_mean / save_invstd / gamma / beta: the ReLU mask of the backward is the decision the
// forward took.  (Two differently rounded expressions, e.g. fmaf((x - mean) * invstd, gamma, beta), disagree in sign for
// pre-activations within a few ulps of zero, and the gradient of such an element is then off by a whole gy entry.)
__device__ __forceinline__ float bn_scale(float gamma, float invstd) { return __fmul_rn(gamma, invstd); }
__device__ __forceinline__ float bn_shift(float mean, float scale, float beta) { return __fmaf_rn(-mean, scale, beta); }
__device__ __forceinline__ float bn_preact(float x, float scale, float shift) { return __fmaf_rn(x, scale, shift); }
// the backward's ReLU test: the gradient passes iff the forward's output was > 0 (a NaN or +-0 output passes none)
__device__ __forceinline__ bool bn_relu_keep(float x, float scale, float shift) { return bn_preact(x, scale, shift) > 0.f; }

// per-column BatchNorm constants from the accumulated sums; `leader` performs the running-statistics side effects
// Every CTA of the consumer runs this for its columns, so it must be cheap: the fp64 part is two multiplies and one FMA (the
// sums are fp64 because E[x^2] - E[x]^2 cancels); the reciprocal square root is taken in fp32 like torch's own BatchNorm
// kernels do.  (fp64 division and square root are software sequences of ~100 instructions each, which would dominate the
// consumer kernel's prologue.)
__device__ __forceinline__ void bn_fold_column(const PgnnBnFold& f, int C, int c, bool leader, float& scale, float& shift) {
  const double s = f.acc[c], ss = f.acc[(int64_t)C + c];
  const double mean = s * f.inv_m;
  double var = fma(ss, f.inv_m, -mean * mean);
  var = var < 0.0 ? 0.0 : var;
  const float invstd = 1.0f / sqrtf((float)var + f.eps);
  const float meanf = (float)mean;
  scale = bn_scale(f.gamma[c], invstd);
  shift = bn_shift(meanf, scale, f.beta[c]);
  if (leader) {
    if (f.save_mean) f.save_mean[c] = meanf;
    if (f.save_invstd) f.save_invstd[c] = invstd;
    if (f.running_mean) f.running_mean[c] = (1.f - f.momentum) * f.running_mean[c] + f.momentum * meanf;
    if (f.running_var) {
      f.running_var[c] = (1.f - f.momentum) * f.running_var[c] + f.momentum * (float)(var * f.unbias);
    }
    if (c == 0 && f.nbt) *f.nbt += 1;
  }
}

// The library's one counter-based hash: the 64-bit key of position `idx` under `seed`.  MaskAtom / MaskEdge / the context root
// draw (transforms.cu, mask_edges.cu, extract.cu) and dropout (below) all draw through it; oracle/step_io_oracle.py and the
// dropout tests restate it.
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t seed, uint64_t idx) {
  uint64_t z = seed + (idx + 1ull) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// Exclusive prefix of one flag across a CTA of kWarps full warps (every thread calls it); the CTA's total in `t`.  `sh` holds
// kWarps ints of shared memory.  The transforms use it to give the selected items of a chunk their output ranks in order.
template <int kWarps>
__device__ __forceinline__ int block_scan_flag(bool a, int* sh, int& t) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, a);
  __syncthreads();
  if (lane == 0) sh[warp] = __popc(m);
  __syncthreads();
  int p = __popc(m & ((1u << lane) - 1u));
  t = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    const int c = sh[w];
    if (w < warp) p += c;
    t += c;
  }
  return p;
}

// one warp: off[0..B] = exclusive scan of f(i)
template <typename F>
__device__ __forceinline__ void warp_scan_to(int64_t B, int64_t* __restrict__ off, F f) {
  const int lane = threadIdx.x & 31;
  int64_t carry = 0;
  for (int64_t base = 0; base < B; base += 32) {
    const int64_t i = base + lane;
    const int64_t n = i < B ? f(i) : 0;
    int64_t s = n;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (i < B) off[i] = carry + s - n;
    carry += __shfl_sync(0xffffffffu, s, 31);
  }
  if (lane == 0) off[B] = carry;
}

// Dropout of layer `layer`'s [rows, C] activation (include/pgnn_b200.h, pgnn_dropout_fwd): element (row i, column c) is kept
// iff (splitmix64(seed, (layer << 40) | (i * C + c)) >> 32) >= thr, and then scaled by `scale`; a dropped element is multiplied
// by 0 (so a dropped NaN / Inf gives NaN, as torch's x * mask * scale does).  The mask is regenerated wherever it is needed
// (forward, backward, on load in the next layer's gather): no mask tensor exists.
struct PgnnDropout {
  float p = 0.f;
  int64_t seed = 0;
  int64_t layer = 0;
  uint64_t thr = 0;   // floor(p * 2^32); 2^32 for p == 1 (no 32-bit draw reaches it: everything is dropped)
  float scale = 1.f;  // (float)(1 / (1 - p)); 0 for p == 1
};

// host: the dropout of (p, seed, layer); false for p outside [0, 1] or NaN
static inline bool pgnn_make_dropout(float p, int64_t seed, int64_t layer, PgnnDropout* d) {
  if (!(p >= 0.f && p <= 1.f)) return false;
  d->p = p;
  d->seed = seed;
  d->layer = layer;
  d->thr = p == 1.f ? (1ull << 32) : (uint64_t)((double)p * 4294967296.0);
  d->scale = p == 1.f ? 0.f : (float)(1.0 / (1.0 - (double)p));
  return true;
}

// the factor element (row, c) of a [*, C] activation is multiplied by: `scale` if kept, else 0
__device__ __forceinline__ float dropout_factor(const PgnnDropout& d, int64_t row, int64_t C, int64_t c) {
  const uint64_t idx = ((uint64_t)d.layer << 40) | (uint64_t)(row * C + c);
  const uint64_t r = splitmix64((uint64_t)d.seed, idx) >> 32;
  return r >= d.thr ? d.scale : 0.f;
}
__device__ __forceinline__ float4 dropout4(float4 v, const PgnnDropout& d, int64_t row, int64_t C, int64_t c) {
  v.x *= dropout_factor(d, row, C, c);
  v.y *= dropout_factor(d, row, C, c + 1);
  v.z *= dropout_factor(d, row, C, c + 2);
  v.w *= dropout_factor(d, row, C, c + 3);
  return v;
}

// Epilogue of the tensor-core GEMM kernel (dense_tc.cu)
struct TcEpilogue {
  const float* bias;      // [N] or null
  int relu;
  const float* mask_src;  // [M,N] (ld = ldm): zero where mask_src <= 0
  int64_t ldm;
  int atomic;             // split-K: accumulate with atomics into a zeroed output
  PgnnGemmHooks hooks;    // fused column reductions over the final output tile (not with split-K)
  int64_t split_stride = 0;  // split-K without atomics: split z stores its tile at C + z * split_stride (folded afterwards)
};

// H100 SXM: 132 SMs.  Grids for grid-stride kernels are sized as a multiple of this.
constexpr int kNumSMs = 132;

// blocks of `threads` for a grid-stride kernel over `items` work items: one item per thread, capped at 16 blocks per SM
static inline int grid_items(int64_t items, int threads) {
  int64_t b = ceil_div(items, threads);
  const int64_t cap = (int64_t)kNumSMs * 16;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// Programmatic dependent launch (PDL).  Every kernel of this library starts with pdl_prologue(): wait until the
// previous kernel in the stream has completed and flushed (griddepcontrol.wait), then allow the NEXT kernel's CTAs to
// become resident (griddepcontrol.launch_dependents) so that its launch latency and prologue overlap this kernel's
// execution; they park on their own wait.  All launches go through pgnn_launch(), which sets the
// programmatic-stream-serialization attribute.  A step is ~85 short kernels: the ~2-3 us of drain + launch between two
// dependent kernels was ~15% of the step.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() {
  pdl_wait();
  pdl_trigger();
}

template <typename... KArgs, typename... Args>
inline cudaError_t pgnn_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const bool prof = g_pgnn_profile_on.load(std::memory_order_relaxed) != 0;
  if (prof) pgnn_profile_mark(reinterpret_cast<const void*>(kernel), st, false);
  const cudaError_t err = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (prof) pgnn_profile_mark(reinterpret_cast<const void*>(kernel), st, true);
  return err;
}

// max(v, 0) that keeps NaN, as torch.relu does (fmaxf(NaN, 0) would return 0 and hide a diverging value)
__device__ __forceinline__ float relu_keep_nan(float v) { return v < 0.f ? 0.f : v; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// The CTA body of a segment mean (global_mean_pool: k_segment_mean_fwd in heads.cu; with kSigmoid, Deep Graph Infomax's summary
// sigmoid(global_mean_pool(x)): k_infomax_summary_fwd in infomax.cu).  One CTA per (segment blockIdx.x, chunk blockIdx.y of 32
// float4 columns): 8 row-lanes (warps) walk the segment's rows eight apart, four independent row loads in flight each, and the
// eight partial sums are folded through shared memory in a fixed order (deterministic).  An empty segment gives the mean 0
// (count.clamp(min=1)).  The first version walked a segment's rows serially in one thread per float4 column: a chain of
// dependent-latency loads that took 258 us for the 64 PPI ego graphs of ~500 nodes of the bio supervised step (a 38 MB read).
template <bool kSigmoid>
__device__ __forceinline__ void segment_mean_cta(const float* __restrict__ x, int64_t ldx, const int* __restrict__ seg_ptr,
                                                 const int* __restrict__ seg_order, int C4, float* __restrict__ out, int64_t ldo) {
  __shared__ float4 red[8][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t b = blockIdx.x;
  const int c4 = blockIdx.y * 32 + lane;
  const int lo = seg_ptr[b], hi = seg_ptr[b + 1];
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c4 < C4) {
    const float* xc = x + 4 * c4;
    auto ld = [&](int k) { return *reinterpret_cast<const float4*>(xc + (int64_t)seg_order[k] * ldx); };
    int k = lo + w;
    for (; k + 24 < hi; k += 32) {
      const float4 v0 = ld(k), v1 = ld(k + 8);
      const float4 v2 = ld(k + 16), v3 = ld(k + 24);
      acc.x += v0.x; acc.y += v0.y; acc.z += v0.z; acc.w += v0.w;
      acc.x += v1.x; acc.y += v1.y; acc.z += v1.z; acc.w += v1.w;
      acc.x += v2.x; acc.y += v2.y; acc.z += v2.z; acc.w += v2.w;
      acc.x += v3.x; acc.y += v3.y; acc.z += v3.z; acc.w += v3.w;
    }
    for (; k < hi; k += 8) {
      const float4 v = ld(k);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  red[w][lane] = acc;
  __syncthreads();
  if (w == 0 && c4 < C4) {
    float4 t = red[0][lane];
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      const float4 v = red[k][lane];
      t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
    }
    const float cnt = (float)max(hi - lo, 1);  // count.clamp(min=1)
    float4 m = make_float4(t.x / cnt, t.y / cnt, t.z / cnt, t.w / cnt);
    if (kSigmoid) {  // torch.sigmoid in fp32: an empty segment gives sigmoid(0) = 0.5
      m.x = 1.f / (1.f + expf(-m.x));
      m.y = 1.f / (1.f + expf(-m.y));
      m.z = 1.f / (1.f + expf(-m.z));
      m.w = 1.f / (1.f + expf(-m.w));
    }
    *reinterpret_cast<float4*>(out + b * ldo + 4 * c4) = m;
  }
}

// edge weight of the aggregation modes (PGNN_AGG_*), for target t with in-degree deg_t (real edges)
__device__ __forceinline__ float agg_weight(int mode, const float* __restrict__ dinv, int t, int s, int deg_t) {
  if (mode == PGNN_AGG_SUM) return 1.0f;
  if (mode == PGNN_AGG_MEAN) return __frcp_rn((float)(deg_t + 1));
  return __fmul_rn(dinv[t], dinv[s]);  // chem/model.py:82
}
