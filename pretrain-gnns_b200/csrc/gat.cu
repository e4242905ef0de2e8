// GAT attention aggregation, forward and backward (chem/model.py:134-165, bio/model.py:147-180).
//
//   x_j' = xl[src] + e_k                                  (chem/model.py:151-152, in-place add)
//   raw  = <att[:, :D], xl[tgt]> + <att[:, D:], x_j'>     (:154)   = p[tgt] + q[src] + r_k
//   a    = softmax_by_target(leaky_relu(raw, slope))      (:156-157; max-subtracted, +1e-16 in the denominator)
//   out  = mean_heads(sum_k a_k x_j') + bias              (:159-165)
//
// The logit splits into per-node scalars p, q (one pass over the nodes) and a per-edge term r_k that only
// depends on the edge FEATURE: with f_k[Q] the feature weights of edge k (chem: one-hot bond type + one-hot
// direction, Q = 9; bio: the 9 attribute bits and a 1 for the bias, Q = 10) and T[Q, H*D] the table /
// transposed encoder, e_k = f_k . T and r_k = f_k . R with R[q,h] = <att[h, D:], T[q, h]> (Q*H scalars).
// Nothing of size [E, H*D] is ever materialised.  One warp owns one target (forward, target-side backward)
// or one source (source-side backward) row; lanes split the D columns for row work and the edges for
// scalar work; no atomics except the handful that fold Q*H scalars.
#include "common.cuh"

#include <cstdlib>

int pgnn_internal_edge_table_bwd(const float* S, int Q, const float* g, int64_t ldg, int64_t g_off, int64_t n, int C, float* gT,
                                 int64_t ldt, cudaStream_t st);
int pgnn_internal_edge_table_bwd_batch(int count, const float* const* S, const int* Q, const float* const* g, const int64_t* ldg,
                                       const int64_t* g_off, float* const* gT, const int64_t* ldt, int64_t n, int C, cudaStream_t st);

namespace {

constexpr int kQ = 10;     // max feature weights per edge
constexpr int kJ = 10;     // columns per lane: D <= 320
constexpr int kMaxH = 4;

template <bool BIO>
__device__ __forceinline__ void edge_feat(const void* __restrict__ feat, int eid, float f[kQ]) {
  if (BIO) {
    if (eid < 0) {
#pragma unroll
      for (int q = 0; q < 9; ++q) f[q] = (q == 7) ? 1.f : 0.f;  // self-loop row (bio/model.py:42-43)
    } else {
      const float* a = reinterpret_cast<const float*>(feat) + (int64_t)eid * 9;
#pragma unroll
      for (int q = 0; q < 9; ++q) f[q] = a[q];
    }
    f[9] = 1.f;  // multiplies the encoder bias row
  } else {
    int a0 = 4, a1 = 0;  // self-loop bond (chem/model.py:42-45)
    if (eid >= 0) {
      const int64_t* a = reinterpret_cast<const int64_t*>(feat) + (int64_t)eid * 2;
      a0 = (int)a[0];
      a1 = (int)a[1];
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) f[q] = (a0 == q) ? 1.f : 0.f;
#pragma unroll
    for (int q = 0; q < 3; ++q) f[6 + q] = (a1 == q) ? 1.f : 0.f;
    f[9] = 0.f;
  }
}

// R[q][h] = <att[h, D:2D], T[q, h*D:(h+1)*D]> into shared memory, one (q,h) pair per warp at a time
__device__ void build_R(const float* __restrict__ att, const float* __restrict__ T, int Q, int H, int D, float* sR) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int p = w; p < Q * H; p += nw) {
    const int q = p / H, h = p % H;
    float s = 0.f;
    for (int c = lane; c < D; c += 32) s = fmaf(att[(int64_t)h * 2 * D + D + c], T[((int64_t)q * H + h) * D + c], s);
    s = warp_sum(s);
    if (lane == 0) sR[q * kMaxH + h] = s;
  }
  __syncthreads();
}

__device__ __forceinline__ float leaky(float v, float slope) { return v > 0.f ? v : v * slope; }

// pq[n][h] = (<att[h,:D], xl[n,h]>, <att[h,D:], xl[n,h]>), one warp per (n, h)
__global__ void __launch_bounds__(256)
k_gat_node_scores(const float* __restrict__ xl, int64_t n, int H, int D, const float* __restrict__ att, float* __restrict__ pq) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t total = n * H;
  for (int64_t w = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); w < total; w += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const int h = (int)(w % H);
    const float* row = xl + w * D;  // [n][h][D] contiguous
    float p = 0.f, q = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float v = row[c];
      p = fmaf(att[(int64_t)h * 2 * D + c], v, p);
      q = fmaf(att[(int64_t)h * 2 * D + D + c], v, q);
    }
    p = warp_sum(p);
    q = warp_sum(q);
    if (lane == 0) {
      pq[w * 2] = p;
      pq[w * 2 + 1] = q;
    }
  }
}

template <bool BIO>
__global__ void __launch_bounds__(256)
k_gat_fwd(const float* __restrict__ xl, int64_t n, int H, int D, const float* __restrict__ att, const float* __restrict__ T,
          const void* __restrict__ feat, const int* __restrict__ rowptr, const int* __restrict__ nbr, const int* __restrict__ eid,
          int64_t E, const float* __restrict__ bias, float slope, const float* __restrict__ pq, float* __restrict__ alpha,
          float* __restrict__ out, int64_t ldo) {
  pdl_prologue();
  constexpr int Q = BIO ? 10 : 9;
  __shared__ float sR[kQ * kMaxH];
  build_R(att, T, Q, H, D, sR);
  const int lane = threadIdx.x & 31;
  const int HD = H * D;
  for (int64_t i = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const int lo = rowptr[i], hi = rowptr[i + 1];
    float oacc[kJ];
#pragma unroll
    for (int j = 0; j < kJ; ++j) oacc[j] = 0.f;
    for (int h = 0; h < H; ++h) {
      const float pi = pq[(i * H + h) * 2];
      // pass 1: segment max of the activated logits (lanes over messages; message hi is the self-loop).  The shift starts
      // from 0, not -inf: torch_geometric 1.0.3's softmax subtracts torch_scatter 1.1.2's scatter_max, whose output is
      // initialised with its default fill_value = 0, i.e. max(0, segment max) (chem/model.py:157).
      float mx = 0.f;
      for (int k = lo + lane; k <= hi; k += 32) {
        const int s = k < hi ? nbr[k] : (int)i;
        float f[kQ];
        edge_feat<BIO>(feat, k < hi ? eid[k] : -1, f);
        float r = 0.f;
#pragma unroll
        for (int q = 0; q < Q; ++q) r = fmaf(f[q], sR[q * kMaxH + h], r);
        mx = fmaxf(mx, leaky(pi + pq[((int64_t)s * H + h) * 2 + 1] + r, slope));
      }
      mx = warp_max(mx);
      // pass 2: exp and segment sum; the un-normalised weights are parked in alpha
      float sum = 0.f;
      for (int k = lo + lane; k <= hi; k += 32) {
        const int s = k < hi ? nbr[k] : (int)i;
        float f[kQ];
        edge_feat<BIO>(feat, k < hi ? eid[k] : -1, f);
        float r = 0.f;
#pragma unroll
        for (int q = 0; q < Q; ++q) r = fmaf(f[q], sR[q * kMaxH + h], r);
        const float ex = expf(leaky(pi + pq[((int64_t)s * H + h) * 2 + 1] + r, slope) - mx);
        alpha[(k < hi ? (int64_t)k : E + i) * H + h] = ex;
        sum += ex;
      }
      sum = warp_sum(sum);
      const float inv = 1.f / (sum + 1e-16f);
      // pass 3: normalise, accumulate the attention-weighted feature summary A[q]
      float A[kQ];
#pragma unroll
      for (int q = 0; q < kQ; ++q) A[q] = 0.f;
      for (int k = lo + lane; k <= hi; k += 32) {
        const int64_t slot = (k < hi ? (int64_t)k : E + i) * H + h;
        const float al = alpha[slot] * inv;
        alpha[slot] = al;
        float f[kQ];
        edge_feat<BIO>(feat, k < hi ? eid[k] : -1, f);
#pragma unroll
        for (int q = 0; q < Q; ++q) A[q] = fmaf(al, f[q], A[q]);
      }
#pragma unroll
      for (int q = 0; q < Q; ++q) A[q] = warp_sum(A[q]);
      __syncwarp();
      // pass 4: rows.  sum_k a_k xl[src_k, h, :]  +  A . T[:, h, :]
      float acc[kJ];
#pragma unroll
      for (int j = 0; j < kJ; ++j) acc[j] = 0.f;
      for (int k = lo; k <= hi; ++k) {
        const int s = k < hi ? nbr[k] : (int)i;
        const float al = alpha[(k < hi ? (int64_t)k : E + i) * H + h];
        const float* row = xl + (int64_t)s * HD + (int64_t)h * D;
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
          const int c = lane + 32 * j;
          if (c < D) acc[j] = fmaf(al, row[c], acc[j]);
        }
      }
      // a molecule node sees 3-5 of the 9 one-hot feature values: rows with A[q] == 0 (warp-uniform, A is warp-reduced) add
      // nothing and are skipped -- the table rows were more than half of this kernel's L1/L2 traffic
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        if (A[q] == 0.f) continue;
        const float* trow = T + (int64_t)q * HD + (int64_t)h * D;
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
          const int c = lane + 32 * j;
          if (c < D) acc[j] = fmaf(A[q], trow[c], acc[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < kJ; ++j) oacc[j] += acc[j];
    }
    const float invH = 1.f / (float)H;
#pragma unroll
    for (int j = 0; j < kJ; ++j) {
      const int c = lane + 32 * j;
      if (c < D) out[i * ldo + c] = oacc[j] * invH + bias[c];
    }
  }
}

// Target-side backward: per target i and head h
//   dal_k = <g_i/H, x_j'>,  dl_k = a_k (dal_k - sum_m a_m dal_m) * leaky'(raw_k)
// writes dl and a indexed by ORIGINAL edge id (self-loop of i at E+i) for the source-side pass, dp[i,h],
// the scaled summary A[h][i][:] (for gT) and folds B[q][h] = sum dl_k f_k[q] into Bsum.
template <bool BIO, int MINB>
__global__ void __launch_bounds__(256, MINB)
k_gat_bwd_target(const float* __restrict__ g, int64_t ldg, const float* __restrict__ xl, int64_t n, int H, int D,
                 const float* __restrict__ att, const float* __restrict__ T, const void* __restrict__ feat,
                 const int* __restrict__ rowptr, const int* __restrict__ nbr, const int* __restrict__ eid, int64_t E, float slope,
                 const float* __restrict__ alpha, const float* __restrict__ pq, float* __restrict__ dl_e, float* __restrict__ al_e,
                 float* __restrict__ dpq, float* __restrict__ Aout, float* __restrict__ Bsum) {
  pdl_prologue();
  constexpr int Q = BIO ? 10 : 9;
  __shared__ float sR[kQ * kMaxH];
  build_R(att, T, Q, H, D, sR);
  const int lane = threadIdx.x & 31;
  const int HD = H * D;
  const float invH = 1.f / (float)H;
  for (int64_t i = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const int lo = rowptr[i], hi = rowptr[i + 1];
    float gi[kJ];
#pragma unroll
    for (int j = 0; j < kJ; ++j) {
      const int c = lane + 32 * j;
      gi[j] = c < D ? g[i * ldg + c] * invH : 0.f;
    }
    // feature columns that any message of this node carries (bit q): GT[q] multiplies f_k[q] only, so the other dot products
    // (each a 300-wide row of T and five shuffles per head) are skipped; a molecule node uses 3-5 of the 9
    unsigned used = 0u;
    for (int k = lo + lane; k <= hi; k += 32) {
      float f[kQ];
      edge_feat<BIO>(feat, k < hi ? eid[k] : -1, f);
#pragma unroll
      for (int q = 0; q < Q; ++q) used |= (f[q] != 0.f) ? (1u << q) : 0u;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) used |= __shfl_xor_sync(0xffffffffu, used, o);
    for (int h = 0; h < H; ++h) {
      float GT[kQ];
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        GT[q] = 0.f;
        if (!((used >> q) & 1u)) continue;
        const float* trow = T + (int64_t)q * HD + (int64_t)h * D;
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
          const int c = lane + 32 * j;
          if (c < D) s = fmaf(gi[j], trow[c], s);
        }
        GT[q] = warp_sum(s);
      }
      // pass A (messages one by one, lanes over columns): dal_k, parked in dl_e; sdot = sum a_k dal_k
      float sdot = 0.f;
      for (int k = lo; k <= hi; ++k) {
        const int s = k < hi ? nbr[k] : (int)i;
        const int e = k < hi ? eid[k] : -1;
        const float* row = xl + (int64_t)s * HD + (int64_t)h * D;
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
          const int c = lane + 32 * j;
          if (c < D) d = fmaf(gi[j], row[c], d);
        }
        d = warp_sum(d);
        float f[kQ];
        edge_feat<BIO>(feat, e, f);
#pragma unroll
        for (int q = 0; q < Q; ++q) d = fmaf(f[q], GT[q], d);
        sdot = fmaf(alpha[(k < hi ? (int64_t)k : E + i) * H + h], d, sdot);
        if (lane == 0) dl_e[(e >= 0 ? (int64_t)e : E + i) * H + h] = d;
      }
      __syncwarp();
      // pass B (lanes over messages): dl_k, dp, A, B
      const float pi = pq[(i * H + h) * 2];
      float dp = 0.f, A[kQ], B[kQ];
#pragma unroll
      for (int q = 0; q < kQ; ++q) A[q] = B[q] = 0.f;
      for (int k = lo + lane; k <= hi; k += 32) {
        const int s = k < hi ? nbr[k] : (int)i;
        const int e = k < hi ? eid[k] : -1;
        const int64_t slot = (e >= 0 ? (int64_t)e : E + i) * H + h;
        float f[kQ];
        edge_feat<BIO>(feat, e, f);
        float r = 0.f;
#pragma unroll
        for (int q = 0; q < Q; ++q) r = fmaf(f[q], sR[q * kMaxH + h], r);
        const float raw = pi + pq[((int64_t)s * H + h) * 2 + 1] + r;
        const float al = alpha[(k < hi ? (int64_t)k : E + i) * H + h];
        const float dl = al * (dl_e[slot] - sdot) * (raw > 0.f ? 1.f : slope);
        dl_e[slot] = dl;
        al_e[slot] = al;
        dp += dl;
#pragma unroll
        for (int q = 0; q < Q; ++q) {
          A[q] = fmaf(al, f[q], A[q]);
          B[q] = fmaf(dl, f[q], B[q]);
        }
      }
      dp = warp_sum(dp);
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        A[q] = warp_sum(A[q]);
        B[q] = warp_sum(B[q]);
      }
      if (lane == 0) {
        dpq[((int64_t)h * n + i) * 2] = dp;
#pragma unroll
        for (int q = 0; q < Q; ++q) {
          Aout[((int64_t)h * n + i) * Q + q] = A[q] * invH;
          if (B[q] != 0.f) atomicAdd(&Bsum[q * kMaxH + h], B[q]);
        }
      }
      __syncwarp();
    }
  }
}

// Source-side backward: gxl[j,h,:] = sum_{k: src=j} a_k g[tgt_k]/H + dq[j,h] att[h,D:] + dp[j,h] att[h,:D]
__global__ void __launch_bounds__(256)
k_gat_bwd_source(const float* __restrict__ g, int64_t ldg, int64_t n, int H, int D, const float* __restrict__ att,
                 const int* __restrict__ rowptr_s, const int* __restrict__ nbr_s, const int* __restrict__ eid_s, int64_t E,
                 const float* __restrict__ dl_e, const float* __restrict__ al_e, float* __restrict__ dpq, float* __restrict__ gxl) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int HD = H * D;
  const float invH = 1.f / (float)H;
  for (int64_t jn = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); jn < n; jn += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const int lo = rowptr_s[jn], hi = rowptr_s[jn + 1];
    for (int h = 0; h < H; ++h) {
      float acc[kJ];
#pragma unroll
      for (int j = 0; j < kJ; ++j) acc[j] = 0.f;
      float dq = 0.f;
      for (int k = lo; k <= hi; ++k) {
        const int64_t t = k < hi ? nbr_s[k] : jn;
        const int64_t slot = (k < hi ? (int64_t)eid_s[k] : E + jn) * H + h;
        const float al = al_e[slot] * invH;
        dq += dl_e[slot];
        const float* row = g + t * ldg;
#pragma unroll
        for (int j = 0; j < kJ; ++j) {
          const int c = lane + 32 * j;
          if (c < D) acc[j] = fmaf(al, row[c], acc[j]);
        }
      }
      const float dp = dpq[((int64_t)h * n + jn) * 2];
#pragma unroll
      for (int j = 0; j < kJ; ++j) {
        const int c = lane + 32 * j;
        if (c < D)
          gxl[jn * HD + (int64_t)h * D + c] = acc[j] + dq * att[(int64_t)h * 2 * D + D + c] + dp * att[(int64_t)h * 2 * D + c];
      }
      if (lane == 0) dpq[((int64_t)h * n + jn) * 2 + 1] = dq;
    }
  }
}

// the r_k = f_k . R path: gatt[h, D:] += sum_q Bsum[q,h] T[q,h,:] ;  gT[q,h,:] += Bsum[q,h] att[h, D:]
__global__ void k_gat_bwd_rterm(const float* __restrict__ Bsum, const float* __restrict__ att, const float* __restrict__ T, int Q,
                                int H, int D, float* __restrict__ gatt, float* __restrict__ gT) {
  pdl_prologue();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * D) return;
  const int h = idx / D, c = idx % D;
  const float aj = att[(int64_t)h * 2 * D + D + c];
  float s = 0.f;
  for (int q = 0; q < Q; ++q) {
    const float b = Bsum[q * kMaxH + h];
    s = fmaf(b, T[((int64_t)q * H + h) * D + c], s);
    gT[((int64_t)q * H + h) * D + c] += b * aj;
  }
  gatt[(int64_t)h * 2 * D + D + c] += s;
}

__global__ void __launch_bounds__(128)
k_colsum_atomic(const float* __restrict__ g, int64_t ld, int64_t M, int N, int rows_per, float* __restrict__ out) {
  pdl_prologue();
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= N) return;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per, r1 = (r0 + rows_per < M) ? r0 + rows_per : M;
  float a = 0.f;
  for (int64_t r = r0; r < r1; ++r) a += g[r * ld + c];
  atomicAdd(&out[c], a);
}

inline int warp_grid(int64_t warps) {
  int64_t b = ceil_div(warps, 8);
  const int64_t cap = (int64_t)kNumSMs * 8;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

struct BwdWs {
  float *dl_e, *al_e, *dpq, *A, *Bsum;
  int64_t bytes;
};
inline BwdWs carve(void* base, int64_t n, int64_t E, int64_t H) {
  char* p = reinterpret_cast<char*>(base);
  BwdWs w;
  int64_t o = 0;
  auto take = [&](int64_t floats) {
    float* r = reinterpret_cast<float*>(p + o);
    o += align_up(floats * 4, 256);
    return r;
  };
  w.dl_e = take((E + n) * H);
  w.al_e = take((E + n) * H);
  w.dpq = take(H * n * 2);
  w.A = take(H * n * kQ);
  w.Bsum = take(kQ * kMaxH);
  w.bytes = o;
  return w;
}

}  // namespace

extern "C" {

int pgnn_gat_fwd(const float* xl, int64_t num_nodes, int64_t H, int64_t D, const float* att, const float* T, int is_bio,
                 const void* feat, const int32_t* rowptr_t, const int32_t* nbr_t, const int32_t* eid_t, int64_t num_edges,
                 const float* bias, float slope, float* alpha, float* pq, float* out, int64_t ldo, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && H > 0 && D > 0 && num_edges >= 0);
  if (H > kMaxH || D > 32 * kJ) return PGNN_EUNSUPPORTED;
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(xl && att && T && rowptr_t && bias && alpha && pq && out && (num_edges == 0 || (feat && nbr_t && eid_t)));
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(pgnn_launch(k_gat_node_scores, dim3(warp_grid(num_nodes * H)), dim3(256), 0, st, xl, num_nodes, (int)H, (int)D, att, pq));
  PGNN_LAUNCH_CHECK();
  if (is_bio)
    PGNN_CUDA(pgnn_launch(k_gat_fwd<true>, dim3(warp_grid(num_nodes)), dim3(256), 0, st, xl, num_nodes, (int)H, (int)D, att, T, feat, rowptr_t, nbr_t, eid_t,
                                                          num_edges, bias, slope, pq, alpha, out, ldo));
  else
    PGNN_CUDA(pgnn_launch(k_gat_fwd<false>, dim3(warp_grid(num_nodes)), dim3(256), 0, st, xl, num_nodes, (int)H, (int)D, att, T, feat, rowptr_t, nbr_t, eid_t,
                                                           num_edges, bias, slope, pq, alpha, out, ldo));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int64_t pgnn_gat_bwd_workspace_bytes(int64_t num_nodes, int64_t num_edges, int64_t H, int64_t D) {
  if (num_nodes < 0 || num_edges < 0 || H <= 0 || D <= 0) return PGNN_EINVAL;
  return carve(nullptr, num_nodes, num_edges, H).bytes;
}

int pgnn_gat_bwd(const float* g, int64_t ldg, const float* xl, int64_t num_nodes, int64_t H, int64_t D, const float* att,
                 const float* T, int is_bio, const void* feat, const int32_t* rowptr_t, const int32_t* nbr_t, const int32_t* eid_t,
                 const int32_t* rowptr_s, const int32_t* nbr_s, const int32_t* eid_s, int64_t num_edges, float slope,
                 const float* alpha, const float* pq, float* gxl, float* gatt, float* gT, float* gbias, void* workspace,
                 int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && H > 0 && D > 0 && num_edges >= 0 && gatt && gT && gbias);
  if (H > kMaxH || D > 32 * kJ) return PGNN_EUNSUPPORTED;
  const int Q = is_bio ? 10 : 9;
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(cudaMemsetAsync(gatt, 0, sizeof(float) * H * 2 * D, st));
  PGNN_CUDA(cudaMemsetAsync(gT, 0, sizeof(float) * Q * H * D, st));
  PGNN_CUDA(cudaMemsetAsync(gbias, 0, sizeof(float) * D, st));
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(g && xl && att && T && rowptr_t && rowptr_s && alpha && pq && gxl && workspace);
  if (workspace_bytes < pgnn_gat_bwd_workspace_bytes(num_nodes, num_edges, H, D)) return PGNN_EWORKSPACE;
  BwdWs w = carve(workspace, num_nodes, num_edges, H);
  PGNN_CUDA(cudaMemsetAsync(w.Bsum, 0, sizeof(float) * kQ * kMaxH, st));
  // PGNN_GAT_OCC=1: the 64-register build (four resident CTAs per SM instead of three; the kernel is a chain of dependent loads per
  // warp, so resident warps are what it is short of); off by default
  static const bool occ4 = getenv("PGNN_GAT_OCC") && getenv("PGNN_GAT_OCC")[0] == '1';
#define PGNN_GAT_BT(BIO_, MINB_)                                                                                                          \
  PGNN_CUDA(pgnn_launch(k_gat_bwd_target<BIO_, MINB_>, dim3(warp_grid(num_nodes)), dim3(256), 0, st, g, ldg, xl, num_nodes, (int)H, (int)D, att, T, \
                        feat, rowptr_t, nbr_t, eid_t, num_edges, slope, alpha, pq, w.dl_e, w.al_e, w.dpq, w.A, w.Bsum))
  if (is_bio) {
    if (occ4) PGNN_GAT_BT(true, 4); else PGNN_GAT_BT(true, 3);
  } else {
    if (occ4) PGNN_GAT_BT(false, 4); else PGNN_GAT_BT(false, 3);
  }
#undef PGNN_GAT_BT
  PGNN_LAUNCH_CHECK();
  PGNN_CUDA(pgnn_launch(k_gat_bwd_source, dim3(warp_grid(num_nodes)), dim3(256), 0, st, g, ldg, num_nodes, (int)H, (int)D, att, rowptr_s, nbr_s, eid_s, num_edges,
                                                         w.dl_e, w.al_e, w.dpq, gxl));
  PGNN_LAUNCH_CHECK();
  // message path into the table: gT[:, h, :] = (A_h / H)^T g;  attention vector: gatt[h, :D] = dp_h^T xl[:, h, :],
  // gatt[h, D:] = dq_h^T xl[:, h, :] -- 2 H reductions over the same rows, batched into one launch when H <= 2
  {
    int batched = PGNN_EUNSUPPORTED;
    if (2 * H <= 4) {
      const float* Sp[4]; const float* gp[4]; float* op[4];
      int Qs[4]; int64_t ldgs[4], goffs[4], ldts[4];
      for (int h = 0; h < (int)H; ++h) {
        Sp[2 * h] = w.A + (int64_t)h * num_nodes * Q; Qs[2 * h] = Q; gp[2 * h] = g; ldgs[2 * h] = ldg; goffs[2 * h] = 0;
        op[2 * h] = gT + (int64_t)h * D; ldts[2 * h] = H * D;
        Sp[2 * h + 1] = w.dpq + (int64_t)h * num_nodes * 2; Qs[2 * h + 1] = 2; gp[2 * h + 1] = xl; ldgs[2 * h + 1] = H * D;
        goffs[2 * h + 1] = (int64_t)h * D; op[2 * h + 1] = gatt + (int64_t)h * 2 * D; ldts[2 * h + 1] = D;
      }
      batched = pgnn_internal_edge_table_bwd_batch((int)(2 * H), Sp, Qs, gp, ldgs, goffs, op, ldts, num_nodes, (int)D, st);
      if (batched != PGNN_OK && batched != PGNN_EUNSUPPORTED) return batched;
    }
    if (batched == PGNN_EUNSUPPORTED) {
      for (int h = 0; h < H; ++h) {
        int rc = pgnn_internal_edge_table_bwd(w.A + (int64_t)h * num_nodes * Q, Q, g, ldg, 0, num_nodes, (int)D, gT + (int64_t)h * D, H * D, st);
        if (rc != PGNN_OK) return rc;
        rc = pgnn_internal_edge_table_bwd(w.dpq + (int64_t)h * num_nodes * 2, 2, xl, H * D, (int64_t)h * D, num_nodes, (int)D,
                                          gatt + (int64_t)h * 2 * D, D, st);
        if (rc != PGNN_OK) return rc;
      }
    }
  }
  PGNN_CUDA(pgnn_launch(k_gat_bwd_rterm, dim3((unsigned)ceil_div(H * D, 128)), dim3(128), 0, st, w.Bsum, att, T, Q, (int)H, (int)D, gatt, gT));
  PGNN_LAUNCH_CHECK();
  {
    int64_t splits = ceil_div(num_nodes, 32);   // ~32 rows per thread (a serial, latency-bound loop): more, shorter row chunks
    if (splits > 512) splits = 512;
    const int rows_per = (int)ceil_div(num_nodes, splits);
    dim3 grid((unsigned)ceil_div(D, 128), (unsigned)ceil_div(num_nodes, rows_per));
    PGNN_CUDA(pgnn_launch(k_colsum_atomic, dim3(grid), dim3(128), 0, st, g, ldg, num_nodes, (int)D, rows_per, gbias));
    PGNN_LAUNCH_CHECK();
  }
  return PGNN_OK;
}

}  // extern "C"
