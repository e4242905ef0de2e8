// Dense node transforms, fp32 FFMA path (precision 0): the torch.nn.Linear calls of GINConv.mlp
// (chem/model.py:29,55; bio/model.py:24,58) and of GCN/SAGE/GAT (chem/model.py:99,147,194), with their
// data- and weight-gradients.  One register-tiled SGEMM template serves the three operand layouts:
//
//   fwd    y[M,N]  = x[M,K]  . w[N,K]^T      A: reduction-contiguous   B: reduction-contiguous
//   dgrad  gx[M,K] = gy[M,N] . w[N,K]        A: reduction-contiguous   B: reduction-strided
//   wgrad  gw[N,K] = gy[M,N]^T . x[M,K]      A: reduction-strided      B: reduction-strided  (split over rows)
//
// This is the exact-fp32 reference path of the library; the tensor-core path (3xTF32 wgmma,
// dense_tc.cu) is checked against it.
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 64, BK = 16, TM = 8, TN = 4;  // 256 threads, 8x4 outputs each

struct Epilogue {
  const float* bias;      // [N] or null
  int relu;               // max(.,0)
  const float* mask_src;  // [M,N] (ld = ldm): multiply by (mask_src > 0)
  int64_t ldm;
  int atomic;             // accumulate with atomicAdd (split-K)
};

template <bool A_RC, bool B_RC>
__global__ void __launch_bounds__(256)
k_sgemm(const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t ldb, float* __restrict__ Cout,
        int64_t ldc, int M, int N, int K, int k_per_split, Epilogue ep) {
  pdl_prologue();
  // element (m, r) of A is A[m*lda + r] if A_RC else A[r*lda + m]; same for B with (n, r)
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);
  const int ty = tid / (BN / TN), tx = tid % (BN / TN);  // 16 x 16
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    // ---- stage A tile [BK][BM] ----
    if (A_RC) {
      // thread -> (row m = tid/4 (+64), 4 consecutive r)
#pragma unroll
      for (int h = 0; h < BM / 64; ++h) {
        const int m = tid / 4 + h * 64, r = (tid % 4) * 4;
        const int gm = m0 + m, gr = k0 + r;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (gm < M) {
          const float* p = A + (int64_t)gm * lda + gr;
          if (gr + 3 < kend && ((lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && ((gr & 3) == 0)) {
            const float4 t = *reinterpret_cast<const float4*>(p);
            v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) if (gr + q < kend) v[q] = p[q];
          }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) As[r + q][m] = v[q];
      }
    } else {
      // thread -> (r = tid/32 (+8), 4 consecutive m at (tid%32)*4)
#pragma unroll
      for (int h = 0; h < BK / 8; ++h) {
        const int r = tid / 32 + h * 8, m = (tid % 32) * 4;
        const int gr = k0 + r, gm = m0 + m;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (gr < kend) {
          const float* p = A + (int64_t)gr * lda + gm;
          if (gm + 3 < M && ((lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && ((gm & 3) == 0)) {
            const float4 t = *reinterpret_cast<const float4*>(p);
            v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) if (gm + q < M) v[q] = p[q];
          }
        }
        *reinterpret_cast<float4*>(&As[r][m]) = make_float4(v[0], v[1], v[2], v[3]);
      }
    }
    // ---- stage B tile [BK][BN] ----
    if (B_RC) {
      const int n = tid / 4, r = (tid % 4) * 4;
      const int gn = n0 + n, gr = k0 + r;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (gn < N) {
        const float* p = B + (int64_t)gn * ldb + gr;
        if (gr + 3 < kend && ((ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0) && ((gr & 3) == 0)) {
          const float4 t = *reinterpret_cast<const float4*>(p);
          v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) if (gr + q < kend) v[q] = p[q];
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) Bs[r + q][n] = v[q];
    } else {
      const int r = tid / 16, n = (tid % 16) * 4;
      const int gr = k0 + r, gn = n0 + n;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (gr < kend) {
        const float* p = B + (int64_t)gr * ldb + gn;
        if (gn + 3 < N && ((ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0) && ((gn & 3) == 0)) {
          const float4 t = *reinterpret_cast<const float4*>(p);
          v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) if (gn + q < N) v[q] = p[q];
        }
      }
      *reinterpret_cast<float4*>(&Bs[r][n]) = make_float4(v[0], v[1], v[2], v[3]);
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < BK; ++r) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[r][ty * TM]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[r][ty * TM + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[r][tx * TN]);
      const float av[TM] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[TN] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  // ---- epilogue ----
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int gm = m0 + ty * TM + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int gn = n0 + tx * TN + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (ep.bias && blockIdx.z == 0) v += ep.bias[gn];
      if (ep.relu) v = relu_keep_nan(v);
      if (ep.mask_src) v = (ep.mask_src[(int64_t)gm * ep.ldm + gn] > 0.f) ? v : 0.f;
      float* dst = Cout + (int64_t)gm * ldc + gn;
      if (ep.atomic) atomicAdd(dst, v); else *dst = v;
    }
  }
}

// gb[n] = sum_m gy[m][n]: grid.x = column tiles of 128, grid.y = row splits, atomics fold the splits.
__global__ void __launch_bounds__(128)
k_colsum(const float* __restrict__ gy, int64_t ld, int M, int N, int rows_per_split, float* __restrict__ gb) {
  pdl_prologue();
  const int n = blockIdx.x * 128 + threadIdx.x;
  if (n >= N) return;
  const int r0 = blockIdx.y * rows_per_split, r1 = min(M, r0 + rows_per_split);
  float a = 0.f;
  for (int r = r0; r < r1; ++r) a += gy[(int64_t)r * ld + n];
  atomicAdd(&gb[n], a);
}

}  // namespace

// tensor-core path (dense_tc.cu); returns PGNN_EUNSUPPORTED when the shape is not covered
int pgnn_tc_linear_fwd(const float*, int64_t, const float*, const float*, int64_t, int64_t, int64_t, int, float*, int64_t,
                       cudaStream_t, const PgnnGemmHooks*);
int pgnn_tc_linear_bwd_x(const float*, int64_t, const float*, int64_t, int64_t, int64_t, const float*, int64_t, float*, int64_t,
                         cudaStream_t, const PgnnGemmHooks*);
int pgnn_tc_linear_bwd_w(const float*, int64_t, const float*, int64_t, int64_t, int64_t, int64_t, float*, float*, cudaStream_t);

extern "C" {

int pgnn_linear_fwd(const float* x, int64_t ldx, const float* w, const float* bias, int64_t M, int64_t N, int64_t K, int relu,
                    float* y, int64_t ldy, int precision, void* stream) {
  PGNN_CHECK_ARG(M >= 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31));
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && w && y && ldx >= K && ldy >= N);
  cudaStream_t st = as_stream(stream);
  if (precision == 1) {
    int rc = pgnn_tc_linear_fwd(x, ldx, w, bias, M, N, K, relu, y, ldy, st, nullptr);
    if (rc != PGNN_EUNSUPPORTED) return rc;
  }
  Epilogue ep{bias, relu, nullptr, 0, 0};
  dim3 grid((unsigned)ceil_div(N, BN), (unsigned)ceil_div(M, BM), 1);
  PGNN_CUDA(pgnn_launch(k_sgemm<true, true>, dim3(grid), dim3(256), 0, st, x, ldx, w, K, y, ldy, (int)M, (int)N, (int)K, (int)K, ep));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_linear_bwd_x(const float* gy, int64_t ldgy, const float* w, int64_t M, int64_t N, int64_t K, const float* relu_src,
                      int64_t ldr, float* gx, int64_t ldgx, int precision, void* stream) {
  PGNN_CHECK_ARG(M >= 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31));
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(gy && w && gx && ldgy >= N && ldgx >= K);
  cudaStream_t st = as_stream(stream);
  if (precision == 1) {
    int rc = pgnn_tc_linear_bwd_x(gy, ldgy, w, M, N, K, relu_src, ldr, gx, ldgx, st, nullptr);
    if (rc != PGNN_EUNSUPPORTED) return rc;
  }
  // out[m, k] = sum_n gy[m, n] * w[n, k]: "N" of the template is K here, reduction runs over N
  Epilogue ep{nullptr, 0, relu_src, ldr, 0};
  dim3 grid((unsigned)ceil_div(K, BN), (unsigned)ceil_div(M, BM), 1);
  PGNN_CUDA(pgnn_launch(k_sgemm<true, false>, dim3(grid), dim3(256), 0, st, gy, ldgy, w, K, gx, ldgx, (int)M, (int)K, (int)N, (int)N, ep));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_linear_bwd_w(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t N, int64_t K, float* gw,
                      float* gb, int precision, void* stream) {
  PGNN_CHECK_ARG(M >= 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31) && gw);
  cudaStream_t st = as_stream(stream);
  if (M == 0) {
    PGNN_CUDA(cudaMemsetAsync(gw, 0, sizeof(float) * N * K, st));
    if (gb) PGNN_CUDA(cudaMemsetAsync(gb, 0, sizeof(float) * N, st));
    return PGNN_OK;
  }
  PGNN_CHECK_ARG(gy && x && ldgy >= N && ldx >= K);
  if (precision == 1) {
    int rc = pgnn_tc_linear_bwd_w(gy, ldgy, x, ldx, M, N, K, gw, gb, st);
    if (rc != PGNN_EUNSUPPORTED) return rc;
  }
  // gw[n, k] = sum_m gy[m, n] * x[m, k]: rows of the output are N, columns K, reduction over the M rows.
  // Few output tiles (N*K is only 600x300), so split the row reduction until the grid covers the SMs twice.
  const int tiles = (int)(ceil_div(N, BM) * ceil_div(K, BN));
  int splits = (int)ceil_div(2 * kNumSMs, tiles);
  const int max_splits = (int)ceil_div(M, 4 * BK);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int per = (int)align_up(ceil_div(M, splits), BK);
  splits = (int)ceil_div(M, per);
  if (splits > 1) PGNN_CUDA(cudaMemsetAsync(gw, 0, sizeof(float) * N * K, st));
  Epilogue ep{nullptr, 0, nullptr, 0, splits > 1};
  dim3 grid((unsigned)ceil_div(K, BN), (unsigned)ceil_div(N, BM), (unsigned)splits);
  PGNN_CUDA(pgnn_launch(k_sgemm<false, false>, dim3(grid), dim3(256), 0, st, gy, ldgy, x, ldx, gw, K, (int)N, (int)K, (int)M, per, ep));
  PGNN_LAUNCH_CHECK();
  if (gb) {
    PGNN_CUDA(cudaMemsetAsync(gb, 0, sizeof(float) * N, st));
    int rsplit = (int)ceil_div(M, 256);
    if (rsplit > 64) rsplit = 64;
    const int rows_per = (int)ceil_div(M, rsplit);
    dim3 g2((unsigned)ceil_div(N, 128), (unsigned)ceil_div(M, rows_per));
    PGNN_CUDA(pgnn_launch(k_colsum, dim3(g2), dim3(128), 0, st, gy, ldgy, (int)M, (int)N, rows_per, gb));
    PGNN_LAUNCH_CHECK();
  }
  return PGNN_OK;
}

}  // extern "C"
