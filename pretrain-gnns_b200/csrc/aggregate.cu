// Neighbour aggregation kernels: the gather + scatter_add of MessagePassing.propagate
// (chem/model.py:49,101,196; bio/model.py:52,111,218) restated as an atomics-free segmented
// reduction over the target-bucketed edge list, plus its transpose and the edge-table gradients.
//
// Work decomposition: one thread per (row, float4 column) item.  D=300 rows are 75 float4, so a
// warp-per-row mapping would idle 21 of 96 lane slots; flattening (row, c4) keeps every lane busy,
// every load is a coalesced 16-byte access into the source row, and bucket metadata (rowptr / nbr)
// is a warp-broadcast load.  Rows are 1200 B, so the whole activation matrix (7 MB at B=256) sits
// in L2 after the first touch; see DESIGN.md for the roofline discussion.
#include "common.cuh"

#include <cstdlib>

namespace {

__device__ __forceinline__ float4 affine_act(float4 v, const float* __restrict__ sc, const float* __restrict__ sh,
                                             int c, int relu) {
  if (sc) {
    const float4 a = ld4(sc + c), b = ld4(sh + c);
    v.x = bn_preact(v.x, a.x, b.x);  // the BatchNorm pre-activation of common.cuh: the backward recomputes it bit for bit
    v.y = bn_preact(v.y, a.y, b.y);
    v.z = bn_preact(v.z, a.z, b.z);
    v.w = bn_preact(v.w, a.w, b.w);
  }
  if (relu) {
    v.x = relu_keep_nan(v.x);
    v.y = relu_keep_nan(v.y);
    v.z = relu_keep_nan(v.z);
    v.w = relu_keep_nan(v.w);
  }
  return v;
}

// acc += w * v with separately rounded multiply and add: keeps the SUM path (w == 1) bit-identical to a
// sequential CPU index_add_ in edge order, which the parity tests exploit.
__device__ __forceinline__ void axpy4(float4& acc, float w, float4 v) {
  acc.x = __fadd_rn(acc.x, __fmul_rn(w, v.x));
  acc.y = __fadd_rn(acc.y, __fmul_rn(w, v.y));
  acc.z = __fadd_rn(acc.z, __fmul_rn(w, v.z));
  acc.w = __fadd_rn(acc.w, __fmul_rn(w, v.w));
}
__device__ __forceinline__ void add4(float4& acc, float4 v) {
  acc.x = __fadd_rn(acc.x, v.x);
  acc.y = __fadd_rn(acc.y, v.y);
  acc.z = __fadd_rn(acc.z, v.z);
  acc.w = __fadd_rn(acc.w, v.w);
}

// DROP: every loaded row j is also multiplied by the dropout mask of (drop.layer, j, c) after the affine + ReLU, i.e. the gather
// reads the previous layer's dropout output without it ever being written (k_aggregate_fwd_drop; k_aggregate_fwd has no mask).
template <bool DROP>
__device__ __forceinline__ void aggregate_fwd_body(const float* __restrict__ x, int64_t ldx, const float* __restrict__ in_scale,
                                                   const float* __restrict__ in_shift, int in_relu, int64_t n, int C4,
                                                   const int* __restrict__ rowptr, const int* __restrict__ nbr, int mode,
                                                   const float* __restrict__ dinv, const float* __restrict__ S, int Q,
                                                   const float* __restrict__ T, const float* __restrict__ T2, int q_split,
                                                   int64_t edge_off, float* __restrict__ out, int64_t ldo, const PgnnBnFold& fold,
                                                   const PgnnDropout& drop) {
  pdl_prologue();
  const int64_t total = n * C4;
  const int C = C4 * 4;
  extern __shared__ __align__(16) float s_aff[];  // [2][C] scale/shift when the producer's BatchNorm is folded in
  if (fold.acc) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) bn_fold_column(fold, C, c, blockIdx.x == 0, s_aff[c], s_aff[C + c]);
    __syncthreads();
    in_scale = s_aff;
    in_shift = s_aff + C;
  }
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / C4);
    const int c = (int)(idx - (int64_t)i * C4) * 4;
    const int lo = rowptr[i], hi = rowptr[i + 1];
    // the effective input row j at columns c..c+3: act(x * in_scale + in_shift), times the mask under DROP
    auto act = [&](float4 v, int j) {
      v = affine_act(v, in_scale, in_shift, c, in_relu);
      if (DROP) v = dropout4(v, drop, j, C, c);
      return v;
    };
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (mode == PGNN_AGG_GCN) {
      const float di = dinv[i];
      for (int k = lo; k < hi; ++k) {
        const int s = nbr[k];
        axpy4(acc, __fmul_rn(di, dinv[s]), act(ld4(x + (int64_t)s * ldx + c), s));
      }
      axpy4(acc, __fmul_rn(di, di), act(ld4(x + (int64_t)i * ldx + c), i));
    } else {
      // the self-loop row and up to four neighbour rows are in flight together (the chain rowptr -> nbr -> row is three
      // dependent L2 round trips per thread: memory-level parallelism, not bandwidth, bounds this kernel); the additions keep
      // the edge order, self-loop last, so the row sums stay bit-identical to a sequential index_add_
      const float4 vself = ld4(x + (int64_t)i * ldx + c);
      int k = lo;
      for (; k + 3 < hi; k += 4) {
        const int s0 = nbr[k], s1 = nbr[k + 1], s2 = nbr[k + 2], s3 = nbr[k + 3];
        const float4 v0 = ld4(x + (int64_t)s0 * ldx + c);
        const float4 v1 = ld4(x + (int64_t)s1 * ldx + c);
        const float4 v2 = ld4(x + (int64_t)s2 * ldx + c);
        const float4 v3 = ld4(x + (int64_t)s3 * ldx + c);
        add4(acc, act(v0, s0));
        add4(acc, act(v1, s1));
        add4(acc, act(v2, s2));
        add4(acc, act(v3, s3));
      }
      if (k + 1 < hi) {
        const int s0 = nbr[k], s1 = nbr[k + 1];
        const float4 v0 = ld4(x + (int64_t)s0 * ldx + c);
        const float4 v1 = ld4(x + (int64_t)s1 * ldx + c);
        add4(acc, act(v0, s0));
        add4(acc, act(v1, s1));
        k += 2;
      }
      if (k < hi) {
        const int s0 = nbr[k];
        add4(acc, act(ld4(x + (int64_t)s0 * ldx + c), s0));
      }
      add4(acc, act(vself, i));  // self-loop last
      if (mode == PGNN_AGG_MEAN) {
        const float cnt = (float)(hi - lo + 1);
        acc.x = __fdiv_rn(acc.x, cnt);
        acc.y = __fdiv_rn(acc.y, cnt);
        acc.z = __fdiv_rn(acc.z, cnt);
        acc.w = __fdiv_rn(acc.w, cnt);
      }
    }
    float4 e = make_float4(0.f, 0.f, 0.f, 0.f);
    if (S) {
      const float* s = S + (int64_t)i * Q;
      for (int q = 0; q < Q; ++q) {
        const float w = s[q];
        if (w == 0.f) continue;  // most of a node's 9-10 summary bins are empty; fmaf(0, t, e) == e, so skipping is exact
        const float4 t = ld4(q < q_split ? T + (int64_t)q * C + c : T2 + (int64_t)(q - q_split) * C + c);
        e.x = fmaf(w, t.x, e.x);
        e.y = fmaf(w, t.y, e.y);
        e.z = fmaf(w, t.z, e.z);
        e.w = fmaf(w, t.w, e.w);
      }
    }
    if (edge_off == 0) {
      add4(acc, e);
      st4(out + (int64_t)i * ldo + c, acc);
    } else {
      st4(out + (int64_t)i * ldo + c, acc);
      st4(out + (int64_t)i * ldo + edge_off + c, e);
    }
  }
}
__global__ void __launch_bounds__(256)
k_aggregate_fwd(const float* __restrict__ x, int64_t ldx, const float* __restrict__ in_scale,
                const float* __restrict__ in_shift, int in_relu, int64_t n, int C4, const int* __restrict__ rowptr,
                const int* __restrict__ nbr, int mode, const float* __restrict__ dinv, const float* __restrict__ S, int Q,
                const float* __restrict__ T, const float* __restrict__ T2, int q_split, int64_t edge_off, float* __restrict__ out,
                int64_t ldo, PgnnBnFold fold) {
  aggregate_fwd_body<false>(x, ldx, in_scale, in_shift, in_relu, n, C4, rowptr, nbr, mode, dinv, S, Q, T, T2, q_split, edge_off, out, ldo,
                            fold, PgnnDropout{});
}
__global__ void __launch_bounds__(256)
k_aggregate_fwd_drop(const float* __restrict__ x, int64_t ldx, const float* __restrict__ in_scale,
                     const float* __restrict__ in_shift, int in_relu, int64_t n, int C4, const int* __restrict__ rowptr,
                     const int* __restrict__ nbr, int mode, const float* __restrict__ dinv, const float* __restrict__ S, int Q,
                     const float* __restrict__ T, const float* __restrict__ T2, int q_split, int64_t edge_off, float* __restrict__ out,
                     int64_t ldo, PgnnBnFold fold, PgnnDropout drop) {
  aggregate_fwd_body<true>(x, ldx, in_scale, in_shift, in_relu, n, C4, rowptr, nbr, mode, dinv, S, Q, T, T2, q_split, edge_off, out, ldo,
                           fold, drop);
}

__global__ void __launch_bounds__(256)
k_aggregate_bwd(const float* __restrict__ g, int64_t ldg, int64_t n, int C4, const int* __restrict__ rowptr_s,
                const int* __restrict__ nbr_s, int mode, const float* __restrict__ dinv, const int* __restrict__ rowptr_t,
                float* __restrict__ gx, int64_t ldgx) {
  pdl_prologue();
  const int64_t total = n * C4;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int j = (int)(idx / C4);
    const int c = (int)(idx - (int64_t)j * C4) * 4;
    const int lo = rowptr_s[j], hi = rowptr_s[j + 1];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (mode == PGNN_AGG_SUM) {
      const float4 vself = ld4(g + (int64_t)j * ldg + c);
      int k = lo;
      for (; k + 3 < hi; k += 4) {
        const int t0 = nbr_s[k], t1 = nbr_s[k + 1], t2 = nbr_s[k + 2], t3 = nbr_s[k + 3];
        const float4 v0 = ld4(g + (int64_t)t0 * ldg + c);
        const float4 v1 = ld4(g + (int64_t)t1 * ldg + c);
        const float4 v2 = ld4(g + (int64_t)t2 * ldg + c);
        const float4 v3 = ld4(g + (int64_t)t3 * ldg + c);
        add4(acc, v0);
        add4(acc, v1);
        add4(acc, v2);
        add4(acc, v3);
      }
      if (k + 1 < hi) {
        const float4 v0 = ld4(g + (int64_t)nbr_s[k] * ldg + c);
        const float4 v1 = ld4(g + (int64_t)nbr_s[k + 1] * ldg + c);
        add4(acc, v0);
        add4(acc, v1);
        k += 2;
      }
      if (k < hi) add4(acc, ld4(g + (int64_t)nbr_s[k] * ldg + c));
      add4(acc, vself);
    } else {
      for (int k = lo; k < hi; ++k) {
        const int t = nbr_s[k];
        const float w = (mode == PGNN_AGG_MEAN) ? __frcp_rn((float)(rowptr_t[t + 1] - rowptr_t[t] + 1))
                                                : __fmul_rn(dinv[t], dinv[j]);
        axpy4(acc, w, ld4(g + (int64_t)t * ldg + c));
      }
      const float wl = (mode == PGNN_AGG_MEAN) ? __frcp_rn((float)(rowptr_t[j + 1] - rowptr_t[j] + 1))
                                               : __fmul_rn(dinv[j], dinv[j]);
      axpy4(acc, wl, ld4(g + (int64_t)j * ldg + c));
    }
    st4(gx + (int64_t)j * ldgx + c, acc);
  }
}

// gT[q][c] = sum_i S[i][q] * g[i][g_off + c].  Blocks of 32 columns x 8 row-lanes sweep 64 rows (8 per thread: the
// per-thread row loop is a chain of dependent-latency loads, 32 rows per thread made the kernel 17 us at N = 6 k) with
// coalesced 128-byte loads; each thread keeps Q register accumulators (S rows are warp-broadcast loads), the 8
// row-lanes are folded in shared memory and one fp32 atomicAdd per (block, q, c) folds the row chunks.
constexpr int kTblRowsSmall = 64, kTblRowsLarge = 256;  // rows per block: small batches are latency-bound, large ones atomics-bound
constexpr int kMaxQ = 16;
__global__ void __launch_bounds__(256)
k_edge_table_bwd(const float* __restrict__ S, int Q, const float* __restrict__ g, int64_t ldg, int64_t g_off, int64_t n,
                 int C, float* __restrict__ gT, int64_t ldt, float* __restrict__ gT2, int q_split, int kTblRows) {
  pdl_prologue();
  __shared__ float red[8][kMaxQ][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = blockIdx.y * 32 + lane;
  const int64_t r0 = (int64_t)blockIdx.x * kTblRows;
  const int64_t r1 = (r0 + kTblRows < n) ? r0 + kTblRows : n;
  float acc[kMaxQ];
#pragma unroll
  for (int q = 0; q < kMaxQ; ++q) acc[q] = 0.f;
  if (c < C) {
#pragma unroll 4
    for (int64_t r = r0 + w; r < r1; r += 8) {
      const float v = g[r * ldg + g_off + c];
      const float* s = S + r * Q;
#pragma unroll
      for (int q = 0; q < kMaxQ; ++q)
        if (q < Q) acc[q] = fmaf(s[q], v, acc[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < kMaxQ; ++q) red[w][q][lane] = acc[q];
  __syncthreads();
  // 256 threads fold (q, lane) pairs: thread t -> q = t / 32 (+8), lane = t % 32
  for (int q = w; q < Q; q += 8) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][q][lane];
    if (c < C) atomicAdd(q < q_split ? &gT[(int64_t)q * ldt + c] : &gT2[(int64_t)(q - q_split) * ldt + c], t);
  }
}

// float4 variant of k_edge_table_bwd: a lane owns FOUR adjacent columns (512-byte warp loads: a quarter of the load instructions
// per byte) and the CTA's S rows are staged in shared memory once (coalesced) instead of Q broadcast loads per row and thread.
// Measured: no faster than the scalar kernel for ONE reduction (the hypothesis that the scalar kernel is load-instruction bound
// was wrong: 58.9 vs 55.6 us at N = 32 k); it is used for the batched form below, where it saves launches.
// 8 row-lanes x 32 column-lanes; the row-lanes are folded through shared memory eight table rows at a time.
// Up to kTblJobs reductions over the same n rows in ONE launch (blockIdx.z): the GAT backward needs four per layer (two heads x
// {message table, attention vector}), each a ~6 us kernel on a molecule batch.
constexpr int kTblJobs = 4;
struct TblJob {
  const float* S;
  const float* g;
  float *gT, *gT2;
  int64_t ldg, g_off, ldt;
  int Q, q_split;
};
struct TblJobs { TblJob j[kTblJobs]; };

template <int ROWS>
__global__ void __launch_bounds__(256)
k_edge_table_bwd_v4(const __grid_constant__ TblJobs jobs, int64_t n, int C4) {
  pdl_prologue();
  const TblJob& job = jobs.j[blockIdx.z];
  const float* __restrict__ S = job.S;
  const float* __restrict__ g = job.g;
  float* __restrict__ gT = job.gT;
  float* __restrict__ gT2 = job.gT2;
  const int64_t ldg = job.ldg, g_off = job.g_off, ldt = job.ldt;
  const int Q = job.Q, q_split = job.q_split;
  __shared__ float sS[ROWS * kMaxQ];
  __shared__ float4 red[8][8][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c4 = blockIdx.y * 32 + lane;
  const int64_t r0 = (int64_t)blockIdx.x * ROWS;
  const int rows = (int)((r0 + ROWS < n) ? ROWS : n - r0);
  for (int i = threadIdx.x; i < rows * Q; i += 256) sS[i] = S[r0 * Q + i];
  __syncthreads();
  float4 acc[kMaxQ];
#pragma unroll
  for (int q = 0; q < kMaxQ; ++q) acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c4 < C4) {
    const float* gp = g + g_off + 4 * c4;
#pragma unroll 4
    for (int r = w; r < rows; r += 8) {
      const float4 v = ld4(gp + (r0 + r) * ldg);
      const float* s = sS + r * Q;
#pragma unroll
      for (int q = 0; q < kMaxQ; ++q)
        if (q < Q) axpy4(acc[q], s[q], v);
    }
  }
#pragma unroll
  for (int pass = 0; pass < kMaxQ / 8; ++pass) {
    if (pass * 8 < Q) {            // uniform across the CTA
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 8; ++q) red[w][q][lane] = acc[pass * 8 + q];
      __syncthreads();
      const int q = pass * 8 + w;  // warp w folds table row pass * 8 + w
      if (q < Q && c4 < C4) {
        float4 t = red[0][w][lane];
#pragma unroll
        for (int k = 1; k < 8; ++k) add4(t, red[k][w][lane]);
        float* dst = (q < q_split ? gT + (int64_t)q * ldt : gT2 + (int64_t)(q - q_split) * ldt) + 4 * c4;
        atomicAdd(dst, t.x);
        atomicAdd(dst + 1, t.y);
        atomicAdd(dst + 2, t.z);
        atomicAdd(dst + 3, t.w);
      }
    }
  }
}

__global__ void __launch_bounds__(256)
k_chem_embed_fwd(const int64_t* __restrict__ x, const float* __restrict__ t1, const float* __restrict__ t2, int64_t n,
                 int C4, int rows1, int rows2, float* __restrict__ out, int64_t ldo, unsigned int* __restrict__ err) {
  pdl_prologue();
  const int64_t total = n * C4;
  const int C = C4 * 4;
  bool bad = false;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / C4;
    const int c = (int)(idx - i * C4) * 4;
    int64_t a0 = x[2 * i], a1 = x[2 * i + 1];
    if (a0 < 0 || a0 >= rows1 || a1 < 0 || a1 >= rows2) {  // nn.Embedding would raise (chem/model.py:231-232): flag, use row 0
      bad = true;
      a0 = (a0 < 0 || a0 >= rows1) ? 0 : a0;
      a1 = (a1 < 0 || a1 >= rows2) ? 0 : a1;
    }
    const float4 a = ld4(t1 + a0 * C + c), b = ld4(t2 + a1 * C + c);
    st4(out + i * ldo + c, make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w)));
  }
  if (bad && err) atomicOr(err, (unsigned)PGNN_DEVERR_ATOM_CODE);
}

// One-hot rows of the two atom codes side by side: oh[i][x0] = 1, oh[i][rows1 + x1] = 1, width padded to a multiple of 4.
// With it the embedding gradient [rows1 + rows2, C] = oh^T . g is a weight-gradient GEMM on the tensor cores (exact products,
// split-K folded in a fixed order: bit-reproducible) instead of N*C/4 vector atomics onto 123 rows (encoder.cu).
__global__ void __launch_bounds__(256)
k_chem_onehot(const int64_t* __restrict__ x, int64_t n, int rows1, int rows2, float* __restrict__ oh, int ld4s) {
  pdl_prologue();
  const int64_t total = n * ld4s;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / ld4s;
    const int c = (int)(idx - i * ld4s) * 4;
    const int64_t a0 = x[2 * i], a1 = x[2 * i + 1];
    const int h0 = (a0 >= 0 && a0 < rows1) ? (int)a0 : -1, h1 = (a1 >= 0 && a1 < rows2) ? rows1 + (int)a1 : -1;
    float4 v;
    v.x = (c == h0 || c == h1) ? 1.f : 0.f;
    v.y = (c + 1 == h0 || c + 1 == h1) ? 1.f : 0.f;
    v.z = (c + 2 == h0 || c + 2 == h1) ? 1.f : 0.f;
    v.w = (c + 3 == h0 || c + 3 == h1) ? 1.f : 0.f;
    st4(oh + idx * 4, v);
  }
}

__global__ void __launch_bounds__(256)
k_chem_embed_bwd(const int64_t* __restrict__ x, const float* __restrict__ g, int64_t ldg, int64_t n, int C4, int rows1, int rows2,
                 float* __restrict__ g1, float* __restrict__ g2) {
  pdl_prologue();
  const int64_t total = n * C4;
  const int C = C4 * 4;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / C4;
    const int c = (int)(idx - i * C4) * 4;
    const float4 v = ld4(g + i * ldg + c);
    const int64_t a0 = x[2 * i], a1 = x[2 * i + 1];  // out-of-range codes were flagged by the forward; they get no gradient
    if (a0 >= 0 && a0 < rows1) atomicAdd(reinterpret_cast<float4*>(g1 + a0 * C + c), v);
    if (a1 >= 0 && a1 < rows2) atomicAdd(reinterpret_cast<float4*>(g2 + a1 * C + c), v);
  }
}

__global__ void __launch_bounds__(256)
k_bio_embed_fwd(const float* __restrict__ x, const float* __restrict__ tab, int64_t n, int C4, float* __restrict__ out,
                int64_t ldo) {
  pdl_prologue();
  const int64_t total = n * C4;
  const int C = C4 * 4;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / C4;
    const int c = (int)(idx - i * C4) * 4;
    st4(out + i * ldo + c, ld4(tab + (int64_t)x[i] * C + c));  // x.to(int64) truncates (bio/model.py:50)
  }
}

// Two table rows only: each thread column-reduces a strided share of the nodes, one atomic per thread.
__global__ void __launch_bounds__(256)
k_bio_embed_bwd(const float* __restrict__ x, const float* __restrict__ g, int64_t ldg, int64_t n, int C,
                float* __restrict__ gtab) {
  pdl_prologue();
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a0 = 0.f, a1 = 0.f;
  for (int64_t i = blockIdx.x; i < n; i += gridDim.x) {
    const float v = g[i * ldg + c];
    if ((int64_t)x[i] == 0) a0 += v; else a1 += v;
  }
  atomicAdd(&gtab[c], a0);
  atomicAdd(&gtab[C + c], a1);
}

}  // namespace

namespace {
bool table_v4_enabled() {
  static const bool on = !(getenv("PGNN_TABLE_V4") && getenv("PGNN_TABLE_V4")[0] == '0');
  return on;
}
int launch_table_v4(const TblJobs& jobs, int count, int64_t n, int C, cudaStream_t st) {
  const int rows = n >= 16384 ? kTblRowsLarge : kTblRowsSmall;
  dim3 grid4((unsigned)ceil_div(n, rows), (unsigned)ceil_div(C / 4, 32), (unsigned)count);
  if (rows == kTblRowsLarge)
    PGNN_CUDA(pgnn_launch(k_edge_table_bwd_v4<kTblRowsLarge>, dim3(grid4), dim3(256), 0, st, jobs, n, C / 4));
  else
    PGNN_CUDA(pgnn_launch(k_edge_table_bwd_v4<kTblRowsSmall>, dim3(grid4), dim3(256), 0, st, jobs, n, C / 4));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}
}  // namespace

// several table reductions over the same n rows and C columns in one launch (count <= 4; every job must meet the float4
// alignment rules, else PGNN_EUNSUPPORTED and the caller issues them one by one)
int pgnn_internal_edge_table_bwd_batch(int count, const float* const* S, const int* Q, const float* const* g, const int64_t* ldg,
                                       const int64_t* g_off, float* const* gT, const int64_t* ldt, int64_t n, int C, cudaStream_t st) {
  if (n == 0 || count == 0) return PGNN_OK;
  if (!table_v4_enabled() || count > kTblJobs || C % 4) return PGNN_EUNSUPPORTED;
  TblJobs jobs{};
  for (int i = 0; i < count; ++i) {
    if (Q[i] > kMaxQ || ldg[i] % 4 || g_off[i] % 4 || !aligned16(g[i])) return PGNN_EUNSUPPORTED;
    jobs.j[i] = TblJob{S[i], g[i], gT[i], nullptr, ldg[i], g_off[i], ldt[i], Q[i], Q[i]};
  }
  return launch_table_v4(jobs, count, n, C, st);
}

// shared with gat.cu / encoder.cu: gT[q*ldt + c] += sum_i S[i][q] g[i][g_off + c]  (caller zeroes gT).
// Rows q >= q_split go to gT2 (the two bond tables of chem/model.py:30-31 are separate parameters).
int pgnn_internal_edge_table_bwd2(const float* S, int Q, const float* g, int64_t ldg, int64_t g_off, int64_t n, int C, float* gT,
                                  int64_t ldt, float* gT2, int q_split, cudaStream_t st) {
  if (n == 0) return PGNN_OK;
  const int rows = n >= 16384 ? kTblRowsLarge : kTblRowsSmall;
  // A single reduction stays on the scalar kernel: the float4 kernel measured no faster alone (bio N = 32 k: 58.9 vs 55.6 us per
  // launch under ncu, 317 vs 296 us per step in the step; GCN: 79 vs 76) -- what it buys is the batching of several reductions
  // into one launch (pgnn_internal_edge_table_bwd_batch, the GAT backward).  PGNN_TABLE_V4=1 forces it here as well.
  static const bool force_v4 = getenv("PGNN_TABLE_V4") && getenv("PGNN_TABLE_V4")[0] == '1';
  if (force_v4 && Q <= kMaxQ && C % 4 == 0 && ldg % 4 == 0 && g_off % 4 == 0 && aligned16(g)) {
    TblJobs jobs{};
    jobs.j[0] = TblJob{S, g, gT, gT2, ldg, g_off, ldt, Q, q_split};
    return launch_table_v4(jobs, 1, n, C, st);
  }
  dim3 grid((unsigned)ceil_div(n, rows), (unsigned)ceil_div(C, 32));
  PGNN_CUDA(pgnn_launch(k_edge_table_bwd, dim3(grid), dim3(256), 0, st, S, Q, g, ldg, g_off, n, C, gT, ldt, gT2, q_split, rows));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}
int pgnn_internal_edge_table_bwd(const float* S, int Q, const float* g, int64_t ldg, int64_t g_off, int64_t n, int C, float* gT,
                                 int64_t ldt, cudaStream_t st) {
  return pgnn_internal_edge_table_bwd2(S, Q, g, ldg, g_off, n, C, gT, ldt, nullptr, Q, st);
}

// aggregate forward with the table given as two row blocks (T rows [0,q_split), T2 rows [q_split,Q))
int pgnn_internal_aggregate_fwd(const float* x, int64_t ldx, const float* in_scale, const float* in_shift, int in_relu,
                                int64_t num_nodes, int64_t C, const int32_t* rowptr_t, const int32_t* nbr_t, int mode, const float* dinv,
                                const float* S, int64_t Q, const float* T, const float* T2, int q_split, int64_t edge_off, float* out,
                                int64_t ldo, cudaStream_t st, const PgnnBnFold* fold, const PgnnDropout* drop) {
  if (num_nodes == 0) return PGNN_OK;
  if (C % 4 || ldx % 4 || ldo % 4 || !aligned16(x) || !aligned16(out) || (T && !aligned16(T)) || (T2 && !aligned16(T2)) ||
      (in_scale && (!aligned16(in_scale) || !aligned16(in_shift))))
    return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  if (drop && drop->p > 0.f)
    PGNN_CUDA(pgnn_launch(k_aggregate_fwd_drop, dim3(grid_items(num_nodes * C4, 256)), dim3(256), fold ? sizeof(float) * 2 * C : 0, st, x, ldx,
                          in_scale, in_shift, in_relu, num_nodes, C4, rowptr_t, nbr_t, mode, dinv, S, (int)Q, T, T2, q_split, edge_off, out,
                          ldo, fold ? *fold : PgnnBnFold{}, *drop));
  else
    PGNN_CUDA(pgnn_launch(k_aggregate_fwd, dim3(grid_items(num_nodes * C4, 256)), dim3(256), fold ? sizeof(float) * 2 * C : 0, st, x, ldx, in_scale,
                          in_shift, in_relu, num_nodes, C4, rowptr_t, nbr_t, mode, dinv, S, (int)Q, T, T2, q_split, edge_off, out, ldo,
                          fold ? *fold : PgnnBnFold{}));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_internal_chem_onehot(const int64_t* x, int64_t n, int rows1, int rows2, float* onehot, int64_t ld, cudaStream_t st) {
  if (n == 0) return PGNN_OK;
  if (ld % 4 || ld < rows1 + rows2 || !aligned16(onehot)) return PGNN_EUNSUPPORTED;
  const int ld4s = (int)(ld / 4);
  PGNN_CUDA(pgnn_launch(k_chem_onehot, dim3(grid_items(n * ld4s, 256)), dim3(256), 0, st, x, n, rows1, rows2, onehot, ld4s));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

extern "C" {

int pgnn_aggregate_fwd(const float* x, int64_t ldx, const float* in_scale, const float* in_shift, int in_relu,
                       int64_t num_nodes, int64_t C, const int32_t* rowptr_t, const int32_t* nbr_t, int mode,
                       const float* dinv, const float* S, int64_t Q, const float* T, int64_t edge_off, float* out, int64_t ldo,
                       void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && C > 0 && mode >= 0 && mode <= 2);
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && rowptr_t && out && (mode != PGNN_AGG_GCN || dinv));
  PGNN_CHECK_ARG((in_scale == nullptr) == (in_shift == nullptr));
  PGNN_CHECK_ARG(!S || (T && Q > 0 && Q <= kMaxQ));
  PGNN_CHECK_ARG(edge_off == 0 || (S && edge_off % 4 == 0));
  return pgnn_internal_aggregate_fwd(x, ldx, in_scale, in_shift, in_relu, num_nodes, C, rowptr_t, nbr_t, mode, dinv, S, Q, T, nullptr,
                                     (int)Q, edge_off, out, ldo, as_stream(stream), nullptr, nullptr);
}

int pgnn_aggregate_bwd(const float* g, int64_t ldg, int64_t num_nodes, int64_t C, const int32_t* rowptr_s,
                       const int32_t* nbr_s, int mode, const float* dinv, const int32_t* rowptr_t, float* gx, int64_t ldgx,
                       void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && C > 0 && mode >= 0 && mode <= 2);
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(g && rowptr_s && gx && (mode != PGNN_AGG_GCN || dinv) && (mode != PGNN_AGG_MEAN || rowptr_t));
  if (C % 4 || ldg % 4 || ldgx % 4 || !aligned16(g) || !aligned16(gx)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_aggregate_bwd, dim3(grid_items(num_nodes * C4, 256)), dim3(256), 0, as_stream(stream), g, ldg, num_nodes, C4, rowptr_s, nbr_s, mode,
                                                                                 dinv, rowptr_t, gx, ldgx));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_edge_table_bwd(const float* S, int64_t Q, const float* g, int64_t ldg, int64_t g_off, int64_t num_nodes, int64_t C,
                        float* gT, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && C > 0 && Q > 0 && Q <= kMaxQ && gT);
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(cudaMemsetAsync(gT, 0, sizeof(float) * Q * C, st));
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(S && g);
  return pgnn_internal_edge_table_bwd(S, (int)Q, g, ldg, g_off, num_nodes, (int)C, gT, C, st);
}

int pgnn_chem_embed_fwd(const int64_t* x, const float* tab1, int64_t rows1, const float* tab2, int64_t rows2, int64_t num_nodes,
                        int64_t C, float* out, int64_t ldo, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && C > 0);
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && tab1 && tab2 && out && rows1 > 0 && rows2 > 0);
  if (C % 4 || ldo % 4 || !aligned16(tab1) || !aligned16(tab2) || !aligned16(out)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_chem_embed_fwd, dim3(grid_items(num_nodes * C4, 256)), dim3(256), 0, as_stream(stream), x, tab1, tab2, num_nodes, C4, (int)rows1, (int)rows2, out, ldo,
                        pgnn_error_flag_ptr()));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_chem_embed_bwd(const int64_t* x, const float* g, int64_t ldg, int64_t num_nodes, int64_t C, float* gtab1,
                        int64_t rows1, float* gtab2, int64_t rows2, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && C > 0 && gtab1 && gtab2 && rows1 > 0 && rows2 > 0);
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(cudaMemsetAsync(gtab1, 0, sizeof(float) * rows1 * C, st));
  PGNN_CUDA(cudaMemsetAsync(gtab2, 0, sizeof(float) * rows2 * C, st));
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && g);
  if (C % 4 || ldg % 4 || !aligned16(g) || !aligned16(gtab1) || !aligned16(gtab2)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_chem_embed_bwd, dim3(grid_items(num_nodes * C4, 256)), dim3(256), 0, st, x, g, ldg, num_nodes, C4, (int)rows1, (int)rows2, gtab1, gtab2));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_bio_embed_fwd(const float* x, const float* tab, int64_t num_nodes, int64_t C, float* out, int64_t ldo, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && C > 0);
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && tab && out);
  if (C % 4 || ldo % 4 || !aligned16(tab) || !aligned16(out)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_bio_embed_fwd, dim3(grid_items(num_nodes * C4, 256)), dim3(256), 0, as_stream(stream), x, tab, num_nodes, C4, out, ldo));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_bio_embed_bwd(const float* x, const float* g, int64_t ldg, int64_t num_nodes, int64_t C, float* gtab, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && C > 0 && gtab);
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(cudaMemsetAsync(gtab, 0, sizeof(float) * 2 * C, st));
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && g);
  // ~32 rows per thread (the row loop is a chain of dependent-latency loads: 64 row blocks took 80 us at N = 32 k)
  int64_t rb = ceil_div(num_nodes, 32);
  if (rb > 4 * kNumSMs) rb = 4 * kNumSMs;
  dim3 grid((unsigned)(rb < 1 ? 1 : rb), (unsigned)ceil_div(C, 256));
  PGNN_CUDA(pgnn_launch(k_bio_embed_bwd, dim3(grid), dim3(256), 0, st, x, g, ldg, num_nodes, (int)C, gtab));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

}  // extern "C"
