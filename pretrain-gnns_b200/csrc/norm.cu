// BatchNorm1d (chem/model.py:252,269; bio/model.py:24), the inter-layer ReLU (bio/model.py:281) and
// GraphSAGE's row L2-normalisation (chem/model.py:201-202), forward and backward.
//
// Column statistics are a grid-wide dependency.  The statistics and backward sweeps walk column tiles: a 256-thread block covers
// 32 * VEC columns (VEC adjacent columns per lane) x 8 row lanes, sweeps row chunks with coalesced loads, accumulates in fp64,
// folds the 8 lanes in shared memory and adds its partial to the [2, C] accumulators with fp64 atomics (order-dependent only at
// the 1e-16 level, i.e. invisible in the fp32 results); a finalize pass over the C columns derives mean / invstd / scale / shift.
// fp64 accumulation makes E[x^2]-E[x]^2 safe (relative error ~1e-16 * mean^2/var).  The backward is the statistics sweep
// (sum(d), sum(d * xhat)) and one apply sweep in the same tiles that writes gx and, for the encoder, the column sums of gx.
//
// Every sweep has two widths: VEC = 4 reads and writes one float4 per lane (C % 4 == 0, row strides multiples of 4, 16-byte
// aligned pointers: the encoder's case), VEC = 1 takes any view.  The sweeps that may carry dropout are templates on DROP as
// well: DROP = true multiplies by the mask of PgnnDropout `drop` (forward: after the ReLU; backward: the incoming gradient, before
// the ReLU mask); DROP = false never reads it.
#include "common.cuh"

#include <initializer_list>

namespace {

// Column tiles: 32 * VEC columns x chunks of tile_rows(VEC) rows.  The float4 tile is 128 columns x 64 rows: every load is a
// 512-byte warp access, 4x fewer instructions than the scalar sweeps and 2 x 8 independent loads in flight per thread.
__host__ __device__ constexpr int tile_cols(int vec) { return 32 * vec; }
__host__ __device__ constexpr int tile_rows(int vec) { return vec == 4 ? 64 : 128; }

// The row sweeps launch one block row per chunk of rows, at most kMaxGridY of them (the limit of gridDim.y): block row y
// handles chunks y, y + gridDim.y, ... in that order, so the fold below has the same structure at every M, and any M < 2^31
// is computed rather than refused at launch.
constexpr int64_t kMaxGridY = 65535;
inline dim3 tile_grid(int vec, int64_t M, int64_t C) {
  const int64_t b = ceil_div(M, tile_rows(vec));
  return dim3((unsigned)ceil_div(C, tile_cols(vec)), (unsigned)(b < kMaxGridY ? b : kMaxGridY));
}

// VEC adjacent floats at p (one 16-byte access for VEC = 4)
template <int VEC>
__device__ __forceinline__ void load_cols(const float* p, float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    const float4 t = ld4(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = *p;
  }
}
template <int VEC>
__device__ __forceinline__ void store_cols(float* p, const float (&v)[VEC]) {
  if constexpr (VEC == 4) st4(p, make_float4(v[0], v[1], v[2], v[3]));
  else *p = v[0];
}

// The column-tile sweeps (k_bn_stats, k_bn_bwd_stats, k_bn_bwd_apply_colsum) share one walk: a lane holds the VEC columns from
// tile_col(), block row y takes the row chunks y, y + gridDim.y, ... of tile_rows(VEC) rows, and warp w the rows r0 + w,
// r0 + w + 8, ... of each chunk.  Each sweep writes that loop around its row body itself: handed to a walker as a lambda, the
// float4 bodies compile to more registers (k_bn_bwd_stats<4, true>: 94 instead of 92).
template <int VEC>
__device__ __forceinline__ int tile_col() { return blockIdx.x * tile_cols(VEC) + (threadIdx.x & 31) * VEC; }

// adds the block's column sums s0, s1 (one partial per row lane) to acc[0][C], acc[1][C]: the 8 lanes are folded in shared memory
// in lane order, then one fp64 atomic per column and sum
template <int VEC>
__device__ __forceinline__ void add_column_pair_sums(const double (&s0)[VEC], const double (&s1)[VEC], int C, double* __restrict__ acc) {
  constexpr int kCols = tile_cols(VEC);
  __shared__ double red[2][8][VEC == 1 ? kCols + 1 : kCols];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < VEC; ++q) {
    red[0][w][lane * VEC + q] = s0[q];
    red[1][w][lane * VEC + q] = s1[q];
  }
  __syncthreads();
  const int which = threadIdx.x / kCols, col = threadIdx.x % kCols;  // thread (which, col) folds sum `which` of tile column col
  if (which < 2 && blockIdx.x * kCols + col < C) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[which][k][col];
    atomicAdd(&acc[(int64_t)which * C + blockIdx.x * kCols + col], t);
  }
}

// the BatchNorm constants of columns c .. c + VEC - 1: the saved statistics, gamma and the forward's scale / shift (bn_preact)
template <int VEC>
struct BnCols {
  float mu[VEC], is[VEC], ga[VEC], sc[VEC], sh[VEC];
  __device__ __forceinline__ void load(const float* mean, const float* invstd, const float* gamma, const float* beta, int c) {
    float be[VEC];
    load_cols<VEC>(mean + c, mu);
    load_cols<VEC>(invstd + c, is);
    load_cols<VEC>(gamma + c, ga);
    load_cols<VEC>(beta + c, be);
#pragma unroll
    for (int q = 0; q < VEC; ++q) {
      sc[q] = bn_scale(ga[q], is[q]);
      sh[q] = bn_shift(mu[q], sc[q], be[q]);
    }
  }
};

// the output of element (r, c) of every forward apply: act(bn_preact(x)), times the dropout mask
template <bool DROP>
__device__ __forceinline__ float bn_out(float x, float sc, float sh, int relu, const PgnnDropout& drop, int64_t r, int64_t C,
                                        int64_t c) {
  float v = bn_preact(x, sc, sh);
  if (relu) v = relu_keep_nan(v);
  if (DROP) v *= dropout_factor(drop, r, C, c);
  return v;
}

template <int VEC>
__global__ void __launch_bounds__(256)
k_bn_stats(const float* __restrict__ x, int64_t ldx, int M, int C, double* __restrict__ acc) {
  pdl_prologue();
  constexpr int kRows = tile_rows(VEC);
  const int c = tile_col<VEC>(), w = threadIdx.x >> 5;
  double s0[VEC] = {}, s1[VEC] = {};
  if (c < C) {
    for (unsigned r0 = blockIdx.y * kRows; r0 < (unsigned)M; r0 += gridDim.y * kRows) {
      const int r1 = (int)min((unsigned)M, r0 + kRows);
#pragma unroll(VEC == 4 ? 8 : 4)  // the float4 sweep unrolls a whole chunk: eight rows per lane
      for (int r = (int)r0 + w; r < r1; r += 8) {
        float v[VEC];
        load_cols<VEC>(x + (int64_t)r * ldx + c, v);
#pragma unroll
        for (int q = 0; q < VEC; ++q) {
          const double u = v[q];
          s0[q] += u;
          s1[q] += u * u;
        }
      }
    }
  }
  add_column_pair_sums<VEC>(s0, s1, C, acc);
}

__global__ void __launch_bounds__(128)
k_bn_finalize(const double* __restrict__ acc, int M, int C, const float* __restrict__ gamma, const float* __restrict__ beta,
              float* __restrict__ running_mean, float* __restrict__ running_var, int64_t* __restrict__ nbt, float momentum,
              float eps, float* __restrict__ save_mean, float* __restrict__ save_invstd, float* __restrict__ scale,
              float* __restrict__ shift) {
  pdl_prologue();
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c == 0 && nbt) *nbt += 1;
  if (c >= C) return;
  const double s = acc[c], ss = acc[(int64_t)C + c];
  const double mean = s / M;
  double var = ss / M - mean * mean;
  var = var < 0.0 ? 0.0 : var;
  const float invstd = (float)(1.0 / sqrt(var + (double)eps));
  const float meanf = (float)mean;
  if (save_mean) save_mean[c] = meanf;
  if (save_invstd) save_invstd[c] = invstd;
  if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * meanf;
  if (running_var) {
    const double unbiased = var * ((double)M / (double)(M > 1 ? M - 1 : 1));
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
  if (scale) {
    const float sc = bn_scale(gamma[c], invstd);
    scale[c] = sc;
    shift[c] = bn_shift(meanf, sc, beta[c]);
  }
}

// y = BatchNorm(x) (+ ReLU) over the M x Cv items of VEC columns
template <int VEC, bool DROP>
__global__ void __launch_bounds__(256)
k_bn_apply(const float* __restrict__ x, int64_t ldx, int64_t M, int Cv, const float* __restrict__ mean,
           const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ beta, int relu,
           float* __restrict__ y, int64_t ldy, PgnnDropout drop) {
  pdl_prologue();
  const int64_t total = M * Cv;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / Cv;
    const int c = (int)(idx - r * Cv) * VEC;
    // (plain arrays rather than a BnCols: with the struct inside the loop, nvcc no longer unrolls it)
    float v[VEC], mu[VEC], is[VEC], ga[VEC], be[VEC];
    load_cols<VEC>(x + r * ldx + c, v);
    load_cols<VEC>(mean + c, mu);
    load_cols<VEC>(invstd + c, is);
    load_cols<VEC>(gamma + c, ga);
    load_cols<VEC>(beta + c, be);
#pragma unroll
    for (int q = 0; q < VEC; ++q) {
      const float sc = bn_scale(ga[q], is[q]);
      v[q] = bn_out<DROP>(v[q], sc, bn_shift(mu[q], sc, be[q]), relu, drop, r, (int64_t)Cv * VEC, (int64_t)c + q);
    }
    store_cols<VEC>(y + r * ldy + c, v);
  }
}

// BatchNorm apply with the finalisation folded in (the last encoder layer materialises node_rep this way)
template <bool DROP>
__global__ void __launch_bounds__(256)
k_bn_apply_fold(const float* __restrict__ x, int64_t ldx, int64_t M, int C, PgnnBnFold fold, int relu, float* __restrict__ y,
                int64_t ldy, PgnnDropout drop) {
  pdl_prologue();
  extern __shared__ __align__(16) float s_aff[];
  for (int c = threadIdx.x; c < C; c += blockDim.x) bn_fold_column(fold, C, c, blockIdx.x == 0, s_aff[c], s_aff[C + c]);
  __syncthreads();
  const int64_t total = M * C;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / C;
    const int c = (int)(idx - r * C);
    y[r * ldy + c] = bn_out<DROP>(x[r * ldx + c], s_aff[c], s_aff[C + c], relu, drop, r, C, c);
  }
}

__global__ void __launch_bounds__(256)
k_bn_eval(const float* __restrict__ x, int64_t ldx, int64_t M, int C, const float* __restrict__ gamma,
          const float* __restrict__ beta, const float* __restrict__ rm, const float* __restrict__ rv, float eps, int relu,
          float* __restrict__ y, int64_t ldy) {
  pdl_prologue();
  const int64_t total = M * C;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / C;
    const int c = (int)(idx - r * C);
    const float invstd = __frcp_rn(__fsqrt_rn(rv[c] + eps));
    float v = fmaf((x[r * ldx + c] - rm[c]) * invstd, gamma[c], beta[c]);
    if (relu) v = relu_keep_nan(v);
    y[r * ldy + c] = v;
  }
}

// sum(d) and sum(d * xhat) per column -> acc[0][C], acc[1][C]
template <int VEC, bool DROP>
__global__ void __launch_bounds__(256)
k_bn_bwd_stats(const float* __restrict__ gy, int64_t ldgy, const float* __restrict__ x, int64_t ldx, int M, int C,
               const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
               const float* __restrict__ invstd, int relu, double* __restrict__ acc, PgnnDropout drop) {
  pdl_prologue();
  constexpr int kRows = tile_rows(VEC);
  const int c = tile_col<VEC>(), w = threadIdx.x >> 5;
  double s0[VEC] = {}, s1[VEC] = {};
  if (c < C) {
    BnCols<VEC> k;  // loaded and derived once per lane, not per row
    k.load(mean, invstd, gamma, beta, c);
    for (unsigned r0 = blockIdx.y * kRows; r0 < (unsigned)M; r0 += gridDim.y * kRows) {
      const int r1 = (int)min((unsigned)M, r0 + kRows);
#pragma unroll 4
      for (int r = (int)r0 + w; r < r1; r += 8) {
        float xv[VEC], g[VEC];
        load_cols<VEC>(x + (int64_t)r * ldx + c, xv);
        load_cols<VEC>(gy + (int64_t)r * ldgy + c, g);
#pragma unroll
        for (int q = 0; q < VEC; ++q) {
          const float xhat = (xv[q] - k.mu[q]) * k.is[q];
          float d = g[q];
          if (DROP) d *= dropout_factor(drop, r, C, c + q);
          if (relu && !bn_relu_keep(xv[q], k.sc[q], k.sh[q])) d = 0.f;
          s0[q] += (double)d;
          s1[q] += (double)d * (double)xhat;  // exact product: small batches make the BN backward a difference of large terms
        }
      }
    }
  }
  add_column_pair_sums<VEC>(s0, s1, C, acc);
}

// gx = gamma * invstd * (d - mean(d) - xhat * mean(d * xhat)) from k_bn_bwd_stats' sums, in the same column tiles, so that the
// column sums of gx (= the bias gradient of the Linear that produced x, chem/model.py:29 mlp[2]) fall out of the same pass when
// colsum is set.  The float4 sweep without dropout keeps three CTAs per SM (80 registers, no spills); the others keep the
// default bound (a minimum of 0 blocks is none), under which the float4 sweep with dropout takes 84 registers.
template <int VEC, bool DROP>
__global__ void __launch_bounds__(256, VEC == 4 && !DROP ? 3 : 0)
k_bn_bwd_apply_colsum(const float* __restrict__ gy, int64_t ldgy, const float* __restrict__ x, int64_t ldx, int M, int C,
                      const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                      const float* __restrict__ invstd, int relu, const double* __restrict__ sums, float* __restrict__ ggamma,
                      float* __restrict__ gbeta, float* __restrict__ gx, int64_t ldgx, float* __restrict__ colsum, PgnnDropout drop) {
  pdl_prologue();
  constexpr int kCols = tile_cols(VEC), kRows = tile_rows(VEC);
  __shared__ float red[8][VEC == 1 ? kCols + 1 : kCols];
  const int c = tile_col<VEC>(), lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float acc[VEC] = {};
  if (c < C) {
    BnCols<VEC> k;
    k.load(mean, invstd, gamma, beta, c);
    float k1[VEC], k2[VEC];
#pragma unroll
    for (int q = 0; q < VEC; ++q) {
      const double sd = sums[c + q], sdx = sums[(int64_t)C + c + q];
      k1[q] = (float)(sd / M);
      k2[q] = (float)(sdx / M);
      if (blockIdx.y == 0 && w == 0) {  // finalisation of the statistics pass folded in
        if (gbeta) gbeta[c + q] = (float)sd;
        if (ggamma) ggamma[c + q] = (float)sdx;
      }
    }
    for (unsigned r0 = blockIdx.y * kRows; r0 < (unsigned)M; r0 += gridDim.y * kRows) {
      const int r1 = (int)min((unsigned)M, r0 + kRows);
#pragma unroll 4
      for (int r = (int)r0 + w; r < r1; r += 8) {
        float xv[VEC], g[VEC], o[VEC];
        load_cols<VEC>(x + (int64_t)r * ldx + c, xv);
        load_cols<VEC>(gy + (int64_t)r * ldgy + c, g);
#pragma unroll
        for (int q = 0; q < VEC; ++q) {
          const float xhat = (xv[q] - k.mu[q]) * k.is[q];
          float d = g[q];
          if (DROP) d *= dropout_factor(drop, r, C, c + q);
          if (relu && !bn_relu_keep(xv[q], k.sc[q], k.sh[q])) d = 0.f;
          o[q] = k.ga[q] * k.is[q] * (d - k1[q] - xhat * k2[q]);
          acc[q] += o[q];
        }
        store_cols<VEC>(gx + (int64_t)r * ldgx + c, o);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < VEC; ++q) red[w][lane * VEC + q] = acc[q];
  __syncthreads();
  if (colsum && threadIdx.x < kCols && blockIdx.x * kCols + threadIdx.x < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
    atomicAdd(&colsum[blockIdx.x * kCols + threadIdx.x], t);
  }
}

// (VEC = 4: one 64-bit division per four elements instead of one per element, and 16-byte accesses.  The scalar kernels ran at
// ~2.5 TB/s on the bio step's [32 k, 300] activations: 180 us per step for four ReLU backward sweeps.)
template <int VEC>
__global__ void __launch_bounds__(256)
k_relu_fwd(const float* __restrict__ x, int64_t ldx, int64_t M, int Cv, float* __restrict__ y, int64_t ldy) {
  pdl_prologue();
  const int64_t total = M * Cv;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / Cv;
    const int c = (int)(idx - r * Cv) * VEC;
    float v[VEC];
    load_cols<VEC>(x + r * ldx + c, v);
#pragma unroll
    for (int q = 0; q < VEC; ++q) v[q] = relu_keep_nan(v[q]);
    store_cols<VEC>(y + r * ldy + c, v);
  }
}
template <int VEC>
__global__ void __launch_bounds__(256)
k_relu_bwd(const float* __restrict__ gy, int64_t ldgy, const float* __restrict__ y, int64_t ldy, int64_t M, int Cv,
           float* __restrict__ gx, int64_t ldgx) {
  pdl_prologue();
  const int64_t total = M * Cv;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / Cv;
    const int c = (int)(idx - r * Cv) * VEC;
    float g[VEC], v[VEC];
    load_cols<VEC>(gy + r * ldgy + c, g);
    load_cols<VEC>(y + r * ldy + c, v);
#pragma unroll
    for (int q = 0; q < VEC; ++q) g[q] = v[q] > 0.f ? g[q] : 0.f;
    store_cols<VEC>(gx + r * ldgx + c, g);
  }
}

// one warp per row
__global__ void __launch_bounds__(256)
k_l2norm_fwd(const float* __restrict__ x, int64_t ldx, int64_t M, int C, float* __restrict__ y, int64_t ldy,
             float* __restrict__ norm) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  for (int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); r < M; r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) { const float v = x[r * ldx + c]; ss = fmaf(v, v, ss); }
    ss = warp_sum(ss);
    const float nrm = fmaxf(sqrtf(ss), 1e-12f);  // F.normalize: x / max(||x||, eps)
    if (lane == 0) norm[r] = nrm;
    for (int c = lane; c < C; c += 32) y[r * ldy + c] = x[r * ldx + c] / nrm;
  }
}
__global__ void __launch_bounds__(256)
k_l2norm_bwd(const float* __restrict__ gy, int64_t ldgy, const float* __restrict__ y, int64_t ldy, const float* __restrict__ norm,
             int64_t M, int C, float* __restrict__ gx, int64_t ldgx) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  for (int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); r < M; r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    float dot = 0.f;
    for (int c = lane; c < C; c += 32) dot = fmaf(gy[r * ldgy + c], y[r * ldy + c], dot);
    dot = warp_sum(dot);
    const float nrm = norm[r];
    // y = x / n with n = max(||x||, eps); for ||x|| > eps: gx = (gy - y * <gy, y>) / n; below eps n is constant
    const bool clamped = nrm <= 1e-12f;
    for (int c = lane; c < C; c += 32) {
      const float g = gy[r * ldgy + c];
      gx[r * ldgx + c] = clamped ? g / nrm : (g - y[r * ldy + c] * dot) / nrm;
    }
  }
}

// The width of the sweeps over a set of [*, C] operands: 4 when their rows hold whole, aligned float4s (C % 4 == 0, every row
// stride a multiple of 4, and every pointer the float4 sweep dereferences 16-byte aligned; a null one is not dereferenced),
// else 1, e.g. for odd C or a view shifted by one float.
int sweep_width(int64_t C, std::initializer_list<int64_t> strides, std::initializer_list<const void*> ptrs) {
  bool v4 = C % 4 == 0;
  for (const int64_t ld : strides) v4 = v4 && ld % 4 == 0;
  for (const void* p : ptrs) v4 = v4 && aligned16(p);
  return v4 ? 4 : 1;
}

// the dropout a caller asked for; none, or p == 0, is inert: the DROP = false kernels run
inline PgnnDropout live(const PgnnDropout* d) { return d && d->p > 0.f ? *d : PgnnDropout{}; }

}  // namespace

// encoder.cu: BatchNorm forward when the column sums / sums of squares were already accumulated (fp64, [2][C]) by the
// epilogue of the GEMM that produced x (PgnnGemmHooks::stats)
// (drop: the mask applied after the ReLU, or null)
int pgnn_internal_bn_apply_fold(const float* x, int64_t ldx, int64_t M, int64_t C, const PgnnBnFold& fold, int relu, float* y,
                                int64_t ldy, cudaStream_t st, const PgnnDropout* drop) {
  const PgnnDropout dr = live(drop);
  PGNN_CUDA(pgnn_launch(dr.p > 0.f ? k_bn_apply_fold<true> : k_bn_apply_fold<false>, dim3(grid_items(M * C, 256)), dim3(256),
                        sizeof(float) * 2 * C, st, x, ldx, M, (int)C, fold, relu, y, ldy, dr));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

// pgnn_bn_fwd_train with the mask `drop` (or null) applied after the ReLU of the materialised y (encoder.cu)
int pgnn_internal_bn_fwd_train(const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma, const float* beta,
                               float* running_mean, float* running_var, int64_t* num_batches_tracked, float momentum, float eps,
                               int relu, float* y, int64_t ldy, float* save_mean, float* save_invstd, float* scale, float* shift,
                               void* workspace, int64_t workspace_bytes, void* stream, const PgnnDropout* drop) {
  PGNN_CHECK_ARG(M > 0 && C > 0 && M < (1ll << 31) && x && gamma && beta && save_mean && save_invstd && workspace);
  PGNN_CHECK_ARG((scale == nullptr) == (shift == nullptr));
  if (workspace_bytes < pgnn_bn_workspace_bytes(M, C)) return PGNN_EWORKSPACE;
  cudaStream_t st = as_stream(stream);
  const PgnnDropout dr = live(drop);
  const bool d = dr.p > 0.f;
  double* acc = reinterpret_cast<double*>(workspace);
  PGNN_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * 2 * C, st));
  const int vec = sweep_width(C, {ldx, y ? ldy : 0}, {x, y, gamma, beta, save_mean, save_invstd});
  PGNN_CUDA(pgnn_launch(vec == 4 ? k_bn_stats<4> : k_bn_stats<1>, tile_grid(vec, M, C), dim3(256), 0, st, x, ldx, (int)M, (int)C, acc));
  PGNN_LAUNCH_CHECK();
  PGNN_CUDA(pgnn_launch(k_bn_finalize, dim3((unsigned)ceil_div(C, 128)), dim3(128), 0, st, acc, (int)M, (int)C, gamma, beta, running_mean, running_var,
                                                           num_batches_tracked, momentum, eps, save_mean, save_invstd, scale,
                                                           shift));
  PGNN_LAUNCH_CHECK();
  if (y) {
    const auto apply = vec == 4 ? (d ? k_bn_apply<4, true> : k_bn_apply<4, false>) : (d ? k_bn_apply<1, true> : k_bn_apply<1, false>);
    PGNN_CUDA(pgnn_launch(apply, dim3(grid_items(M * (C / vec), 256)), dim3(256), 0, st, x, ldx, M, (int)(C / vec), save_mean, save_invstd,
                          gamma, beta, relu, y, ldy, dr));
    PGNN_LAUNCH_CHECK();
  }
  return PGNN_OK;
}

// pgnn_bn_bwd with the forward's mask `drop` (or null) applied to gy before the ReLU mask, which also leaves the column sums of gx
// in colsum[C] (OVERWRITTEN) when colsum is set (encoder.cu)
int pgnn_internal_bn_bwd(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma,
                         const float* beta, const float* save_mean, const float* save_invstd, int relu, float* gx, int64_t ldgx,
                         float* ggamma, float* gbeta, float* colsum, void* workspace, int64_t workspace_bytes, cudaStream_t st,
                         const PgnnDropout* drop) {
  PGNN_CHECK_ARG(M > 0 && C > 0 && M < (1ll << 31) && gy && x && gamma && beta && save_mean && save_invstd && gx && workspace);
  if (workspace_bytes < pgnn_bn_workspace_bytes(M, C)) return PGNN_EWORKSPACE;
  const PgnnDropout dr = live(drop);
  const bool d = dr.p > 0.f;
  double* acc = reinterpret_cast<double*>(workspace);
  PGNN_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * 2 * C, st));
  if (colsum) PGNN_CUDA(cudaMemsetAsync(colsum, 0, sizeof(float) * C, st));
  const int vec = sweep_width(C, {ldgy, ldx, ldgx}, {gy, x, gx, gamma, beta, save_mean, save_invstd});
  const dim3 grid = tile_grid(vec, M, C);
  const auto stats = vec == 4 ? (d ? k_bn_bwd_stats<4, true> : k_bn_bwd_stats<4, false>)
                              : (d ? k_bn_bwd_stats<1, true> : k_bn_bwd_stats<1, false>);
  PGNN_CUDA(pgnn_launch(stats, grid, dim3(256), 0, st, gy, ldgy, x, ldx, (int)M, (int)C, gamma, beta, save_mean, save_invstd, relu, acc, dr));
  PGNN_LAUNCH_CHECK();
  const auto apply = vec == 4 ? (d ? k_bn_bwd_apply_colsum<4, true> : k_bn_bwd_apply_colsum<4, false>)
                              : (d ? k_bn_bwd_apply_colsum<1, true> : k_bn_bwd_apply_colsum<1, false>);
  PGNN_CUDA(pgnn_launch(apply, grid, dim3(256), 0, st, gy, ldgy, x, ldx, (int)M, (int)C, gamma, beta, save_mean, save_invstd, relu,
                        (const double*)acc, ggamma, gbeta, gx, ldgx, colsum, dr));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

extern "C" {

int64_t pgnn_bn_workspace_bytes(int64_t M, int64_t C) {
  if (M < 0 || C <= 0) return PGNN_EINVAL;
  return align_up(2 * C * 8, 256);
}

int pgnn_bn_fwd_train(const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma, const float* beta,
                      float* running_mean, float* running_var, int64_t* num_batches_tracked, float momentum, float eps, int relu,
                      float* y, int64_t ldy, float* save_mean, float* save_invstd, float* scale, float* shift, void* workspace,
                      int64_t workspace_bytes, void* stream) {
  return pgnn_internal_bn_fwd_train(x, ldx, M, C, gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps, relu, y, ldy,
                                    save_mean, save_invstd, scale, shift, workspace, workspace_bytes, stream, nullptr);
}

int pgnn_bn_fwd_eval(const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma, const float* beta,
                     const float* running_mean, const float* running_var, float eps, int relu, float* y, int64_t ldy,
                     void* stream) {
  PGNN_CHECK_ARG(M >= 0 && C > 0);
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && gamma && beta && running_mean && running_var && y);
  PGNN_CUDA(pgnn_launch(k_bn_eval, dim3(grid_items(M * C, 256)), dim3(256), 0, as_stream(stream), x, ldx, M, (int)C, gamma, beta, running_mean, running_var, eps,
                                                                    relu, y, ldy));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_bn_bwd(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma,
                const float* beta, const float* save_mean, const float* save_invstd, int relu, float* gx, int64_t ldgx,
                float* ggamma, float* gbeta, void* workspace, int64_t workspace_bytes, void* stream) {
  return pgnn_internal_bn_bwd(gy, ldgy, x, ldx, M, C, gamma, beta, save_mean, save_invstd, relu, gx, ldgx, ggamma, gbeta, nullptr,
                              workspace, workspace_bytes, as_stream(stream), nullptr);
}

int pgnn_relu_fwd(const float* x, int64_t ldx, int64_t M, int64_t C, float* y, int64_t ldy, void* stream) {
  PGNN_CHECK_ARG(M >= 0 && C > 0);
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && y);
  const int vec = sweep_width(C, {ldx, ldy}, {x, y});
  PGNN_CUDA(pgnn_launch(vec == 4 ? k_relu_fwd<4> : k_relu_fwd<1>, dim3(grid_items(M * (C / vec), 256)), dim3(256), 0, as_stream(stream), x,
                        ldx, M, (int)(C / vec), y, ldy));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_relu_bwd(const float* gy, int64_t ldgy, const float* y, int64_t ldy_, int64_t M, int64_t C, float* gx, int64_t ldgx,
                  void* stream) {
  PGNN_CHECK_ARG(M >= 0 && C > 0);
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(gy && y && gx);
  const int vec = sweep_width(C, {ldgy, ldy_, ldgx}, {gy, y, gx});
  PGNN_CUDA(pgnn_launch(vec == 4 ? k_relu_bwd<4> : k_relu_bwd<1>, dim3(grid_items(M * (C / vec), 256)), dim3(256), 0, as_stream(stream), gy,
                        ldgy, y, ldy_, M, (int)(C / vec), gx, ldgx));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_l2norm_fwd(const float* x, int64_t ldx, int64_t M, int64_t C, float* y, int64_t ldy, float* norm, void* stream) {
  PGNN_CHECK_ARG(M >= 0 && C > 0);
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && y && norm);
  PGNN_CUDA(pgnn_launch(k_l2norm_fwd, dim3(grid_items(M * 32, 256)), dim3(256), 0, as_stream(stream), x, ldx, M, (int)C, y, ldy, norm));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_l2norm_bwd(const float* gy, int64_t ldgy, const float* y, int64_t ldy_, const float* norm, int64_t M, int64_t C,
                    float* gx, int64_t ldgx, void* stream) {
  PGNN_CHECK_ARG(M >= 0 && C > 0);
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(gy && y && norm && gx);
  PGNN_CUDA(pgnn_launch(k_l2norm_bwd, dim3(grid_items(M * 32, 256)), dim3(256), 0, as_stream(stream), gy, ldgy, y, ldy_, norm, M, (int)C, gx, ldgx));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_debug_bn_apply_fold(const float* x, int64_t ldx, int64_t M, int64_t C, const double* sums, const float* gamma, const float* beta,
                             float* running_mean, float* running_var, int64_t* num_batches_tracked, float momentum, float eps,
                             float* save_mean, float* save_invstd, int relu, float* y, int64_t ldy, float drop_p, int64_t drop_seed,
                             int64_t drop_layer, void* stream) {
  PGNN_CHECK_ARG(M > 0 && C > 0 && M < (1ll << 31) && C <= 6144 && x && sums && gamma && beta && y && ldx >= C && ldy >= C);
  PgnnDropout drop;
  PGNN_CHECK_ARG(pgnn_make_dropout(drop_p, drop_seed, drop_layer, &drop));
  PgnnBnFold fold;
  fold.acc = sums; fold.gamma = gamma; fold.beta = beta;
  fold.running_mean = running_mean; fold.running_var = running_var; fold.nbt = num_batches_tracked;
  fold.save_mean = save_mean; fold.save_invstd = save_invstd;
  fold.momentum = momentum; fold.eps = eps; fold.set_rows((int)M);
  return pgnn_internal_bn_apply_fold(x, ldx, M, C, fold, relu, y, ldy, as_stream(stream), &drop);
}

int pgnn_debug_bn_bwd_colsum(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma,
                             const float* beta, const float* save_mean, const float* save_invstd, int relu, float* gx, int64_t ldgx,
                             float* ggamma, float* gbeta, float* colsum, float drop_p, int64_t drop_seed, int64_t drop_layer,
                             void* workspace, int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(M > 0 && C > 0 && M < (1ll << 31) && gy && x && gamma && beta && save_mean && save_invstd && gx && colsum && workspace);
  PGNN_CHECK_ARG(ldgy >= C && ldx >= C && ldgx >= C);
  PgnnDropout drop;
  PGNN_CHECK_ARG(pgnn_make_dropout(drop_p, drop_seed, drop_layer, &drop));
  return pgnn_internal_bn_bwd(gy, ldgy, x, ldx, M, C, gamma, beta, save_mean, save_invstd, relu, gx, ldgx, ggamma, gbeta, colsum,
                              workspace, workspace_bytes, as_stream(stream), &drop);
}

}  // extern "C"
