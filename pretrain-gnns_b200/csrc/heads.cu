// Graph-level and self-supervised heads: global_mean_pool (chem/model.py:326,369; bio/model.py:342),
// row gathers for masked atoms / bonds / centre nodes (chem/pretrain_masking.py:51,58-59;
// chem/pretrain_contextpred.py:54,57; bio/model.py:343) and the cyclic-shift negative-sampling dot
// products (chem/pretrain_contextpred.py:36-39,64-67).
#include "common.cuh"

namespace {

// global_mean_pool: the segment-mean body of common.cuh (segment_mean_cta), shared with Deep Graph Infomax's summary.
__global__ void __launch_bounds__(256)
k_segment_mean_fwd(const float* __restrict__ x, int64_t ldx, const int* __restrict__ seg_ptr, const int* __restrict__ seg_order,
                   int64_t num_seg, int C4, float* __restrict__ out, int64_t ldo) {
  pdl_prologue();
  segment_mean_cta<false>(x, ldx, seg_ptr, seg_order, C4, out, ldo);
}

__global__ void __launch_bounds__(256)
k_segment_mean_bwd(const float* __restrict__ g, int64_t ldg, const int64_t* __restrict__ seg, const int* __restrict__ seg_ptr,
                   int64_t n, int C4, float* __restrict__ gx, int64_t ldgx) {
  pdl_prologue();
  const int64_t total = n * C4;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / C4;
    const int c = (int)(idx - r * C4) * 4;
    const int64_t b = seg[r];
    const float cnt = (float)max(seg_ptr[b + 1] - seg_ptr[b], 1);
    const float4 v = ld4(g + b * ldg + c);
    st4(gx + r * ldgx + c, make_float4(v.x / cnt, v.y / cnt, v.z / cnt, v.w / cnt));
  }
}

__global__ void __launch_bounds__(256)
k_row_gather_fwd(const float* __restrict__ x, int64_t ldx, int64_t rows, const int64_t* __restrict__ idx1, const int64_t* __restrict__ idx2,
                 int64_t m, int C4, float* __restrict__ out, int64_t ldo, unsigned int* __restrict__ err) {
  pdl_prologue();
  const int64_t total = m * C4;
  bool bad = false;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / C4;
    const int c = (int)(idx - r * C4) * 4;
    const int64_t i1 = idx1[r], i2 = idx2 ? idx2[r] : 0;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);  // an out-of-range index (torch would assert) contributes zeros and is flagged
    if (i1 >= 0 && i1 < rows) v = ld4(x + i1 * ldx + c); else bad = true;
    if (idx2) {
      if (i2 >= 0 && i2 < rows) {
        const float4 u = ld4(x + i2 * ldx + c);
        v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
      } else {
        bad = true;
      }
    }
    st4(out + r * ldo + c, v);
  }
  if (bad && err) atomicOr(err, (unsigned)PGNN_DEVERR_GATHER);
}

// index_put_(accumulate=True): duplicates are legal (two masked bonds may share an atom), so rows are
// accumulated with vector atomics (red.global.add.v4.f32).
__global__ void __launch_bounds__(256)
k_row_gather_bwd(const float* __restrict__ g, int64_t ldg, const int64_t* __restrict__ idx1, const int64_t* __restrict__ idx2,
                 int64_t m, int C4, float* __restrict__ gx, int64_t ldgx, int64_t rows) {
  pdl_prologue();
  const int64_t total = m * C4;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / C4;
    const int c = (int)(idx - r * C4) * 4;
    const float4 v = ld4(g + r * ldg + c);
    const int64_t i1 = idx1[r];
    if (i1 >= 0 && i1 < rows) atomicAdd(reinterpret_cast<float4*>(gx + i1 * ldgx + c), v);
    if (idx2) {
      const int64_t i2 = idx2[r];
      if (i2 >= 0 && i2 < rows) atomicAdd(reinterpret_cast<float4*>(gx + i2 * ldgx + c), v);
    }
  }
}

// one warp per row
__global__ void __launch_bounds__(256)
k_shifted_rowdot_fwd(const float* __restrict__ a, int64_t lda, const float* __restrict__ b, int64_t ldb, int64_t B, int C,
                     int64_t shift, float* __restrict__ out) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  for (int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); r < B; r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const int64_t rb = (r + shift) % B;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(a[r * lda + c], b[rb * ldb + c], s);
    s = warp_sum(s);
    if (lane == 0) out[r] = s;
  }
}

__global__ void __launch_bounds__(256)
k_shifted_rowdot_bwd(const float* __restrict__ g, const float* __restrict__ a, int64_t lda, const float* __restrict__ b,
                     int64_t ldb, int64_t B, int C, int64_t shift, int accumulate, float* __restrict__ ga, int64_t ldga,
                     float* __restrict__ gb, int64_t ldgb) {
  pdl_prologue();
  const int64_t total = B * C;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / C;
    const int c = (int)(idx - r * C);
    const int64_t rf = (r + shift) % B;            // partner row of a[r]
    const int64_t rbk = ((r - shift) % B + B) % B;  // row of a whose partner is b[r]
    const float va = g[r] * b[rf * ldb + c];
    const float vb = g[rbk] * a[rbk * lda + c];
    if (accumulate) {
      ga[r * ldga + c] += va;
      gb[r * ldgb + c] += vb;
    } else {
      ga[r * ldga + c] = va;
      gb[r * ldgb + c] = vb;
    }
  }
}

// Mean cross-entropy over fp32 logits evaluated in fp64, as `criterion(pred_node.double(), labels)` does
// (chem/pretrain_masking.py:26,52).  One warp per row: max, log-sum-exp, -log p[label]; the same pass writes
// dlogits = (softmax - onehot) / M, so the backward of the loss needs no kernel of its own.
__global__ void __launch_bounds__(256)
k_softmax_ce(const float* __restrict__ logits, int64_t ld, int64_t M, int V, const int64_t* __restrict__ labels,
             double* __restrict__ loss_mean, float* __restrict__ dlogits, int64_t lddl, unsigned int* __restrict__ err) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  for (int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); r < M; r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const float* row = logits + r * ld;
    double mx = -1e300;
    for (int v = lane; v < V; v += 32) mx = fmax(mx, (double)row[v]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    double se = 0.0;
    for (int v = lane; v < V; v += 32) se += exp((double)row[v] - mx);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    const double lse = mx + log(se);
    int64_t y = labels[r];
    if (y < 0 || y >= V) {  // nll_loss would assert: flag, and let the row contribute log-sum-exp only
      if (lane == 0 && err) atomicOr(err, (unsigned)PGNN_DEVERR_LABEL);
      y = -1;
    }
    const double inv_m = 1.0 / (double)M;
    for (int v = lane; v < V; v += 32) {
      const double p = exp((double)row[v] - lse);
      dlogits[r * lddl + v] = (float)((p - (v == y ? 1.0 : 0.0)) * inv_m);
    }
    for (int v = V + lane; v < lddl; v += 32) dlogits[r * lddl + v] = 0.f;  // padding columns of the 16-byte-aligned row
    if (lane == 0) atomicAdd(loss_mean, (lse - (y >= 0 ? (double)row[y] : 0.0)) * inv_m);
  }
}

// The same loss with the class of row m given as a row of Q floats: label = the first index of the row's maximum, what
// `torch.argmax(batch.mask_edge_label, dim=1)` computes for bio masking (bio/pretrain_masking.py:47-55; torch >= 1.7 documents
// the first maximal index).  That head has V = 7 and ~10^5 rows per step, so a row is held by a group of G lanes (the
// power of two >= V, at most 32; 32 / G rows per warp) instead of a whole warp, and the loss is folded deterministically: one
// fp64 partial per CTA, summed in CTA order by the last CTA to finish (the ticket scheme of losses.cu), no floating-point atomics.
// A label >= V, or a label row without a finite maximum (a NaN in it, a +-Inf maximum), sets PGNN_DEVERR_LABEL and the row
// contributes as a bad int64 label does in k_softmax_ce: its log-sum-exp only.
constexpr int kCeRowsThreads = 256;
constexpr int kCeRowsMaxBlocks = kNumSMs * 4;

struct CeRowsWs {
  double partial[kCeRowsMaxBlocks];
  unsigned int ticket;
  unsigned int pad;
};

template <int G>
__global__ void __launch_bounds__(kCeRowsThreads)
k_softmax_ce_rows(const float* __restrict__ logits, int64_t ld, int64_t M, int V, const float* __restrict__ lab, int64_t ldl, int Q,
                  CeRowsWs* __restrict__ ws, double* __restrict__ loss_mean, float* __restrict__ dlogits, int64_t lddl,
                  unsigned int* __restrict__ err) {
  pdl_prologue();
  constexpr int kRowsPerCta = kCeRowsThreads / G;
  __shared__ double s_part[kCeRowsThreads / 32];
  __shared__ bool s_last;
  const int sub = threadIdx.x & (G - 1);
  const double inv_m = 1.0 / (double)M;
  double acc = 0.0;
  bool bad = false;
  // `base` is uniform across the CTA, so every lane of a warp runs every iteration and the group shuffles below may use the
  // full mask; the lanes of a row past M (`live` false) only take part in the shuffles
  for (int64_t base = (int64_t)blockIdx.x * kRowsPerCta; base < M; base += (int64_t)gridDim.x * kRowsPerCta) {
    const int64_t r = base + threadIdx.x / G;
    const bool live = r < M;
    const float* row = logits + r * ld;
    double mx = -1e300;
    if (live)
      for (int v = sub; v < V; v += G) mx = fmax(mx, (double)row[v]);
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    double se = 0.0;
    if (live)
      for (int v = sub; v < V; v += G) se += exp((double)row[v] - mx);
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    const double lse = mx + log(se);
    float best = -INFINITY;
    int bi = Q, nan = 0;
    if (live) {
      const float* t = lab + r * ldl;
      for (int q = sub; q < Q; q += G) {  // ascending per lane: a lane keeps its first maximum
        const float x = t[q];
        if (x != x) nan = 1;
        else if (x > best) best = x, bi = q;
      }
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      nan |= __shfl_xor_sync(0xffffffffu, nan, o);
      if (ob > best || (ob == best && oi < bi)) best = ob, bi = oi;
    }
    int y = bi;
    if (nan || !isfinite(best) || y >= V) {
      bad |= live;
      y = -1;
    }
    if (live) {
      for (int v = sub; v < V; v += G) {
        const double p = exp((double)row[v] - lse);
        dlogits[r * lddl + v] = (float)((p - (v == y ? 1.0 : 0.0)) * inv_m);
      }
      for (int v = V + sub; v < lddl; v += G) dlogits[r * lddl + v] = 0.f;  // padding columns of the 16-byte-aligned row
      if (sub == 0) acc += lse - (y >= 0 ? (double)row[y] : 0.0);
    }
  }
  if (bad && err) atomicOr(err, (unsigned)PGNN_DEVERR_LABEL);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int w = 0; w < kCeRowsThreads / 32; ++w) b += s_part[w];
    ws->partial[blockIdx.x] = b;
    __threadfence();
    s_last = atomicAdd(&ws->ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    double s = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) s += reinterpret_cast<volatile double*>(ws->partial)[b];
    *loss_mean = s * inv_m;
  }
}

// Edge prediction (chem/pretrain_edgepred.py:31-41, bio/pretrain_edgepred.py): pos_p = <x[u_p], x[v_p]> over the P positive
// pairs, neg_q likewise over the Q negative ones, loss = mean_p BCE(pos_p, 1) + mean_q BCE(neg_q, 0).  A pair is held by 8 lanes
// over float4 columns: lane l sums columns 4l, 4l+32, ... with fmaf in that order, and the 8 lane sums are folded by a fixed
// xor-shuffle tree (deterministic).  The BCE terms and d loss / d score = (sigmoid(s) - t) / P (or / Q) are evaluated in fp64;
// the loss is folded as k_softmax_ce_rows folds it (per-CTA fp64 partials summed in CTA order by the last CTA).  An empty side
// gives torch's mean over nothing, NaN, and no gradient.  The same pass writes the P + Q pairs as one contiguous [2, P + Q]
// list for pgnn_graph_prep, which buckets them for the backward.
constexpr int kPairThreads = 256;
constexpr int kPairsPerCta = kPairThreads / 8;
constexpr int kPairMaxBlocks = kNumSMs * 8;

struct PairBceWs {
  double partial[2][kPairMaxBlocks];
  unsigned int ticket;
  unsigned int pad;
};

__global__ void __launch_bounds__(kPairThreads)
k_edge_pair_bce_fwd(const float* __restrict__ x, int64_t ldx, int64_t N, int C4, const int64_t* __restrict__ pu, const int64_t* __restrict__ pv,
                    int64_t ps, int64_t P, const int64_t* __restrict__ qu, const int64_t* __restrict__ qv, int64_t qs, int64_t Q,
                    PairBceWs* __restrict__ ws, double* __restrict__ loss, float* __restrict__ pos, float* __restrict__ neg,
                    float* __restrict__ dscore, int64_t* __restrict__ pairs, unsigned int* __restrict__ err) {
  pdl_prologue();
  __shared__ double s_part[2][kPairThreads / 32];
  __shared__ bool s_last;
  const int sub = threadIdx.x & 7;
  const int64_t total = P + Q;
  double acc[2] = {0.0, 0.0};
  bool bad = false;
  // `base` is uniform across the CTA: every lane runs every iteration and takes part in the group shuffles
  for (int64_t base = (int64_t)blockIdx.x * kPairsPerCta; base < total; base += (int64_t)gridDim.x * kPairsPerCta) {
    const int64_t p = base + (threadIdx.x >> 3);
    const bool live = p < total, is_neg = p >= P;
    int64_t u = 0, v = 0;
    if (live) {
      if (is_neg) u = qu[(p - P) * qs], v = qv[(p - P) * qs];
      else u = pu[p * ps], v = pv[p * ps];
    }
    const bool ok = live && u >= 0 && u < N && v >= 0 && v < N;   // a pair outside [0, N) scores 0 and is flagged
    float s = 0.f;
    if (ok) {
      const float* xu = x + u * ldx;
      const float* xv = x + v * ldx;
      for (int c = sub; c < C4; c += 8) {
        const float4 a = ld4(xu + 4 * c), b = ld4(xv + 4 * c);
        s = fmaf(a.x, b.x, s);
        s = fmaf(a.y, b.y, s);
        s = fmaf(a.z, b.z, s);
        s = fmaf(a.w, b.w, s);
      }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (live && sub == 0) {
      bad |= !ok;
      const double xs = (double)s, t = is_neg ? 0.0 : 1.0;
      const double e = exp(-fabs(xs));
      const double sig = xs >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);
      acc[is_neg] += fmax(xs, 0.0) - xs * t + log1p(e);
      dscore[p] = (float)((sig - t) / (double)(is_neg ? Q : P));
      if (is_neg) neg[p - P] = s;
      else pos[p] = s;
      pairs[p] = u;
      pairs[total + p] = v;
    }
  }
  if (bad && err) atomicOr(err, (unsigned)PGNN_DEVERR_GATHER);
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    double a = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if ((threadIdx.x & 31) == 0) s_part[k][threadIdx.x >> 5] = a;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double b0 = 0.0, b1 = 0.0;
    for (int w = 0; w < kPairThreads / 32; ++w) b0 += s_part[0][w], b1 += s_part[1][w];
    ws->partial[0][blockIdx.x] = b0;
    ws->partial[1][blockIdx.x] = b1;
    __threadfence();
    s_last = atomicAdd(&ws->ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    __threadfence();
    double sp = 0.0, sq = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) {
      sp += reinterpret_cast<volatile double*>(ws->partial[0])[b];
      sq += reinterpret_cast<volatile double*>(ws->partial[1])[b];
    }
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    *loss = (P > 0 ? sp / (double)P : nan) + (Q > 0 ? sq / (double)Q : nan);
  }
}

// d x[i] = sum_{p: u_p = i} g_p x[v_p] + sum_{p: v_p = i} g_p x[u_p],  g_p = dscore[p] * (float)*gscale, each sum over the pairs
// in pair order (the stable buckets of pgnn_graph_prep over the [2, P + Q] pair list: _t by u with payload v, _s by v with payload
// u).  One thread per (row, float4 column), fmaf accumulation, no atomics: deterministic.  A pair with u = v sits in both buckets
// of its row and contributes 2 g x[u].
__global__ void __launch_bounds__(256)
k_edge_pair_bce_bwd(const float* __restrict__ x, int64_t ldx, int64_t N, int C4, const float* __restrict__ dscore,
                    const double* __restrict__ gscale, const int* __restrict__ rowptr_t, const int* __restrict__ nbr_t,
                    const int* __restrict__ eid_t, const int* __restrict__ rowptr_s, const int* __restrict__ nbr_s,
                    const int* __restrict__ eid_s, float* __restrict__ gx, int64_t ldgx) {
  pdl_prologue();
  const float gs = (float)*gscale;
  const int64_t total = N * C4;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / C4;
    const int c = (int)(idx - i * C4) * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      const int* rowptr = side ? rowptr_s : rowptr_t;
      const int* nbr = side ? nbr_s : nbr_t;
      const int* eid = side ? eid_s : eid_t;
      const int lo = rowptr[i], hi = rowptr[i + 1];
#pragma unroll 4
      for (int k = lo; k < hi; ++k) {
        const float g = __fmul_rn(dscore[eid[k]], gs);
        const float4 v = ld4(x + (int64_t)nbr[k] * ldx + c);
        acc.x = fmaf(g, v.x, acc.x);
        acc.y = fmaf(g, v.y, acc.y);
        acc.z = fmaf(g, v.z, acc.z);
        acc.w = fmaf(g, v.w, acc.w);
      }
    }
    st4(gx + i * ldgx + c, acc);
  }
}

}  // namespace

extern "C" {

int pgnn_segment_mean_fwd(const float* x, int64_t ldx, const int32_t* seg_ptr, const int32_t* seg_order, int64_t num_seg,
                          int64_t C, float* out, int64_t ldo, void* stream) {
  PGNN_CHECK_ARG(num_seg >= 0 && C > 0);
  if (num_seg == 0) return PGNN_OK;
  PGNN_CHECK_ARG(seg_ptr && out);
  if (C % 4 || ldx % 4 || ldo % 4 || !aligned16(x) || !aligned16(out)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_segment_mean_fwd, dim3((unsigned)num_seg, (unsigned)ceil_div(C4, 32)), dim3(256), 0, as_stream(stream), x, ldx, seg_ptr, seg_order,
                        num_seg, C4, out, ldo));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_segment_mean_bwd(const float* g, int64_t ldg, const int64_t* seg, const int32_t* seg_ptr, int64_t num_rows, int64_t C,
                          float* gx, int64_t ldgx, void* stream) {
  PGNN_CHECK_ARG(num_rows >= 0 && C > 0);
  if (num_rows == 0) return PGNN_OK;
  PGNN_CHECK_ARG(g && seg && seg_ptr && gx);
  if (C % 4 || ldg % 4 || ldgx % 4 || !aligned16(g) || !aligned16(gx)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_segment_mean_bwd, dim3(grid_items(num_rows * C4, 256)), dim3(256), 0, as_stream(stream), g, ldg, seg, seg_ptr, num_rows, C4, gx, ldgx));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_row_gather_fwd(const float* x, int64_t ldx, int64_t num_rows, const int64_t* idx, const int64_t* idx2, int64_t num_idx, int64_t C,
                        float* out, int64_t ldo, void* stream) {
  PGNN_CHECK_ARG(num_idx >= 0 && C > 0 && num_rows >= 0);
  if (num_idx == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && idx && out);
  if (C % 4 || ldx % 4 || ldo % 4 || !aligned16(x) || !aligned16(out)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_row_gather_fwd, dim3(grid_items(num_idx * C4, 256)), dim3(256), 0, as_stream(stream), x, ldx, num_rows, idx, idx2, num_idx, C4, out, ldo,
                        pgnn_error_flag_ptr()));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_row_gather_bwd(const float* g, int64_t ldg, const int64_t* idx, const int64_t* idx2, int64_t num_idx, int64_t C,
                        float* gx, int64_t ldgx, int64_t num_rows, void* stream) {
  PGNN_CHECK_ARG(num_idx >= 0 && C > 0);
  if (num_idx == 0) return PGNN_OK;
  PGNN_CHECK_ARG(g && idx && gx);
  if (C % 4 || ldg % 4 || ldgx % 4 || !aligned16(g) || !aligned16(gx)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_row_gather_bwd, dim3(grid_items(num_idx * C4, 256)), dim3(256), 0, as_stream(stream), g, ldg, idx, idx2, num_idx, C4, gx, ldgx, num_rows));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_softmax_ce_fwd(const float* logits, int64_t ld, int64_t M, int64_t V, const int64_t* labels, double* loss_mean,
                        float* dlogits, int64_t lddl, void* stream) {
  PGNN_CHECK_ARG(M >= 0 && V > 0 && loss_mean && lddl >= V && ld >= V);
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(cudaMemsetAsync(loss_mean, 0, sizeof(double), st));
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(logits && labels && dlogits);
  PGNN_CUDA(pgnn_launch(k_softmax_ce, dim3(grid_items(M * 32, 256)), dim3(256), 0, st, logits, ld, M, (int)V, labels, loss_mean, dlogits, lddl, pgnn_error_flag_ptr()));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int64_t pgnn_softmax_ce_rows_workspace_bytes(void) { return (int64_t)sizeof(CeRowsWs); }

int pgnn_softmax_ce_rows_fwd(const float* logits, int64_t ld, int64_t M, int64_t V, const float* label_rows, int64_t ld_label, int64_t Q,
                             double* loss_mean, float* dlogits, int64_t lddl, void* workspace, int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(M >= 0 && V > 0 && V <= (1 << 30) && Q > 0 && Q <= (1 << 30) && loss_mean && lddl >= V && ld >= V && ld_label >= Q && workspace);
  if (workspace_bytes < (int64_t)sizeof(CeRowsWs)) return PGNN_EWORKSPACE;
  cudaStream_t st = as_stream(stream);
  if (M == 0) {
    PGNN_CUDA(cudaMemsetAsync(loss_mean, 0, sizeof(double), st));
    return PGNN_OK;
  }
  PGNN_CHECK_ARG(logits && label_rows && dlogits);
  CeRowsWs* ws = reinterpret_cast<CeRowsWs*>(workspace);
  PGNN_CUDA(cudaMemsetAsync(&ws->ticket, 0, sizeof(unsigned int), st));
  const int G = V <= 1 ? 1 : V <= 2 ? 2 : V <= 4 ? 4 : V <= 8 ? 8 : V <= 16 ? 16 : 32;
  int64_t blocks = ceil_div(M, (int64_t)(kCeRowsThreads / G));
  if (blocks > kCeRowsMaxBlocks) blocks = kCeRowsMaxBlocks;
  const dim3 grid((unsigned)blocks), block(kCeRowsThreads);
  unsigned int* err = pgnn_error_flag_ptr();
#define PGNN_CE_ROWS(g) pgnn_launch(k_softmax_ce_rows<g>, grid, block, 0, st, logits, ld, M, (int)V, label_rows, ld_label, (int)Q, ws, loss_mean, \
                                    dlogits, lddl, err)
  switch (G) {
    case 1: PGNN_CUDA(PGNN_CE_ROWS(1)); break;
    case 2: PGNN_CUDA(PGNN_CE_ROWS(2)); break;
    case 4: PGNN_CUDA(PGNN_CE_ROWS(4)); break;
    case 8: PGNN_CUDA(PGNN_CE_ROWS(8)); break;
    case 16: PGNN_CUDA(PGNN_CE_ROWS(16)); break;
    default: PGNN_CUDA(PGNN_CE_ROWS(32)); break;
  }
#undef PGNN_CE_ROWS
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int64_t pgnn_edge_pair_bce_workspace_bytes(void) { return (int64_t)sizeof(PairBceWs); }

int pgnn_edge_pair_bce_fwd(const float* x, int64_t ldx, int64_t N, int64_t C, const int64_t* pos_u, const int64_t* pos_v, int64_t pos_stride,
                           int64_t P, const int64_t* neg_u, const int64_t* neg_v, int64_t neg_stride, int64_t Q, double* loss,
                           float* pos_scores, float* neg_scores, float* dscore, int64_t* pairs, void* workspace, int64_t workspace_bytes,
                           void* stream) {
  PGNN_CHECK_ARG(N >= 0 && C > 0 && ldx >= C && P >= 0 && Q >= 0 && loss && workspace);
  PGNN_CHECK_ARG(P == 0 || (pos_u && pos_v && pos_scores));
  PGNN_CHECK_ARG(Q == 0 || (neg_u && neg_v && neg_scores));
  PGNN_CHECK_ARG(P + Q == 0 || (x && dscore && pairs));
  if (workspace_bytes < (int64_t)sizeof(PairBceWs)) return PGNN_EWORKSPACE;
  if (C % 4 || ldx % 4 || (x && !aligned16(x))) return PGNN_EUNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  PairBceWs* ws = reinterpret_cast<PairBceWs*>(workspace);
  PGNN_CUDA(cudaMemsetAsync(&ws->ticket, 0, sizeof(unsigned int), st));
  int64_t blocks = ceil_div(P + Q, (int64_t)kPairsPerCta);
  if (blocks > kPairMaxBlocks) blocks = kPairMaxBlocks;
  if (blocks < 1) blocks = 1;   // one CTA writes the loss of an empty batch (NaN)
  PGNN_CUDA(pgnn_launch(k_edge_pair_bce_fwd, dim3((unsigned)blocks), dim3(kPairThreads), 0, st, x, ldx, N, (int)(C / 4), pos_u, pos_v, pos_stride,
                        P, neg_u, neg_v, neg_stride, Q, ws, loss, pos_scores, neg_scores, dscore, pairs, pgnn_error_flag_ptr()));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_edge_pair_bce_bwd(const float* x, int64_t ldx, int64_t N, int64_t C, const float* dscore, const double* gscale,
                           const int32_t* rowptr_t, const int32_t* nbr_t, const int32_t* eid_t, const int32_t* rowptr_s,
                           const int32_t* nbr_s, const int32_t* eid_s, float* gx, int64_t ldgx, void* stream) {
  PGNN_CHECK_ARG(N >= 0 && C > 0 && ldx >= C && ldgx >= C);
  if (N == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && gscale && rowptr_t && rowptr_s && gx);
  if (C % 4 || ldx % 4 || ldgx % 4 || !aligned16(x) || !aligned16(gx)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_edge_pair_bce_bwd, dim3(grid_items(N * C4, 256)), dim3(256), 0, as_stream(stream), x, ldx, N, C4, dscore, gscale,
                        rowptr_t, nbr_t, eid_t, rowptr_s, nbr_s, eid_s, gx, ldgx));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_shifted_rowdot_fwd(const float* a, int64_t lda, const float* b, int64_t ldb, int64_t B, int64_t C, int64_t shift,
                            float* out, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && C > 0 && shift >= 0);
  if (B == 0) return PGNN_OK;
  PGNN_CHECK_ARG(a && b && out);
  PGNN_CUDA(pgnn_launch(k_shifted_rowdot_fwd, dim3(grid_items(B * 32, 256)), dim3(256), 0, as_stream(stream), a, lda, b, ldb, B, (int)C, shift, out));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_shifted_rowdot_bwd(const float* g, const float* a, int64_t lda, const float* b, int64_t ldb, int64_t B, int64_t C,
                            int64_t shift, int accumulate, float* ga, int64_t ldga, float* gb, int64_t ldgb, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && C > 0 && shift >= 0);
  if (B == 0) return PGNN_OK;
  PGNN_CHECK_ARG(g && a && b && ga && gb);
  PGNN_CUDA(pgnn_launch(k_shifted_rowdot_bwd, dim3(grid_items(B * C, 256)), dim3(256), 0, as_stream(stream), g, a, lda, b, ldb, B, (int)C, shift, accumulate, ga,
                                                                             ldga, gb, ldgb));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

}  // extern "C"
