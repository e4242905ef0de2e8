// Deep Graph Infomax head (chem/pretrain_deepgraphinfomax.py:61-73, bio/pretrain_deepgraphinfomax.py alike):
//   S = sigmoid(global_mean_pool(x, batch))                       [G, C]
//   H = S . W                                                     [G, C]  (Discriminator: h = summary @ weight)
//   pos_i = <x_i, H[b_i]>,  neg_i = <x_i, H[(b_i + 1) mod G]>     (cycle_index(G, 1) shifts the summaries by one graph)
//   loss = mean_i BCE(pos_i, 1) + mean_i BCE(neg_i, 0)
// The three G x C x C products are the library's GEMM entry points (pgnn_linear_*); the kernels here are the summary, the fused
// scores + BCE pass, the per-graph reduction of the backward and its node pass.  No N x C temporary exists in either direction.
#include "common.cuh"

// the 3xTF32 weight-gradient GEMM with a split-K partials workspace (dense_tc.cu): its splits are folded in order, so dW repeats
// bit for bit (pgnn_linear_bwd_w folds them with atomics)
int pgnn_tc_linear_bwd_w_ws(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t N, int64_t K, float* gw,
                            float* gb, float* partials, int64_t partial_floats, cudaStream_t st);
int64_t pgnn_tc_wgrad_workspace_floats(int64_t M, int64_t N, int64_t K);

namespace {

__global__ void __launch_bounds__(256)
k_infomax_summary_fwd(const float* __restrict__ x, int64_t ldx, const int* __restrict__ seg_ptr, const int* __restrict__ seg_order,
                      int C4, float* __restrict__ S, int64_t lds) {
  pdl_prologue();
  segment_mean_cta<true>(x, ldx, seg_ptr, seg_order, C4, S, lds);
}

// Scores + BCE.  A node is held by 8 lanes over float4 columns: lane l sums columns 4l, 4l+32, ... of both products with fmaf in
// that order, and the 8 lane sums are folded by a fixed xor-shuffle tree (deterministic).  x_i is read once for both scores; the
// G summary rows H stay in L2.  The BCE terms and d loss / d score ((sigmoid - 1) / N, sigmoid / N) are evaluated in fp64 and the
// loss is folded from per-CTA fp64 partials in CTA order by the last CTA, as k_edge_pair_bce_fwd folds it.  N = 0 gives torch's
// mean over nothing, NaN.  A graph id outside [0, G) (pgnn_bucket has flagged it while building the segments) scores 0 and reads
// nothing.
constexpr int kImxThreads = 256;
constexpr int kImxNodesPerCta = kImxThreads / 8;
constexpr int kImxMaxBlocks = kNumSMs * 8;

struct InfomaxBceWs {
  double partial[2][kImxMaxBlocks];
  unsigned int ticket;
  unsigned int pad;
};

__global__ void __launch_bounds__(kImxThreads)
k_infomax_bce_fwd(const float* __restrict__ x, int64_t ldx, int64_t N, int C4, const int64_t* __restrict__ batch, int64_t G,
                  const float* __restrict__ H, InfomaxBceWs* __restrict__ ws, double* __restrict__ loss, float* __restrict__ pos,
                  float* __restrict__ neg, float* __restrict__ dscore) {
  pdl_prologue();
  __shared__ double s_part[2][kImxThreads / 32];
  __shared__ bool s_last;
  const int sub = threadIdx.x & 7;
  double acc[2] = {0.0, 0.0};
  // `base` is uniform across the CTA: every lane runs every iteration and takes part in the group shuffles
  for (int64_t base = (int64_t)blockIdx.x * kImxNodesPerCta; base < N; base += (int64_t)gridDim.x * kImxNodesPerCta) {
    const int64_t i = base + (threadIdx.x >> 3);
    const bool live = i < N;
    const int64_t g = live ? batch[i] : 0;
    float sp = 0.f, sn = 0.f;
    if (live && g >= 0 && g < G) {
      const int64_t gn = g + 1 == G ? 0 : g + 1;
      const float* xi = x + i * ldx;
      const float* hp = H + g * 4 * C4;
      const float* hn = H + gn * 4 * C4;
      for (int c = sub; c < C4; c += 8) {
        const float4 a = ld4(xi + 4 * c), p = ld4(hp + 4 * c), q = ld4(hn + 4 * c);
        sp = fmaf(a.x, p.x, sp);
        sp = fmaf(a.y, p.y, sp);
        sp = fmaf(a.z, p.z, sp);
        sp = fmaf(a.w, p.w, sp);
        sn = fmaf(a.x, q.x, sn);
        sn = fmaf(a.y, q.y, sn);
        sn = fmaf(a.z, q.z, sn);
        sn = fmaf(a.w, q.w, sn);
      }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      sp += __shfl_xor_sync(0xffffffffu, sp, o);
      sn += __shfl_xor_sync(0xffffffffu, sn, o);
    }
    if (live && sub == 0) {
      const double xp = (double)sp, xn = (double)sn;
      const double ep = exp(-fabs(xp)), en = exp(-fabs(xn));
      const double sigp = xp >= 0.0 ? 1.0 / (1.0 + ep) : ep / (1.0 + ep);
      const double sign = xn >= 0.0 ? 1.0 / (1.0 + en) : en / (1.0 + en);
      acc[0] += fmax(xp, 0.0) - xp + log1p(ep);
      acc[1] += fmax(xn, 0.0) + log1p(en);
      dscore[i] = (float)((sigp - 1.0) / (double)N);
      dscore[N + i] = (float)(sign / (double)N);
      pos[i] = sp;
      neg[i] = sn;
    }
  }
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
    for (int w = 0; w < kImxThreads / 32; ++w) b0 += s_part[0][w], b1 += s_part[1][w];
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
    *loss = N > 0 ? sp / (double)N + sq / (double)N : nan;
  }
}

// Per-graph reduction of the backward: dH[g] = gscale * (sum_{i in g} dpos_i x_i + sum_{i in prev(g)} dneg_i x_i), prev(g) =
// (g - 1) mod G.  One CTA per (graph, chunk of 32 float4 columns), the layout of segment_mean_cta: warp w takes the rows
// lo + w, lo + w + 8, ... of graph g (weight dpos), then those of prev(g) (weight dneg), in the segments' stable order, with an
// fmaf chain; the 8 partials are folded in warp order through shared memory.  No atomics: deterministic, and a 500-row bio graph
// is 8 chains of ~60 rows instead of one of 500.
__global__ void __launch_bounds__(256)
k_infomax_graph_reduce(const float* __restrict__ x, int64_t ldx, int64_t N, int C4, const int* __restrict__ seg_ptr,
                       const int* __restrict__ seg_order, int64_t G, const float* __restrict__ dscore, const double* __restrict__ gscale,
                       float* __restrict__ dH) {
  pdl_prologue();
  __shared__ float4 red[8][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t g = blockIdx.x;
  const int64_t gp = g == 0 ? G - 1 : g - 1;
  const int c4 = blockIdx.y * 32 + lane;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c4 < C4) {
    const float* xc = x + 4 * c4;
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      const int64_t s = side ? gp : g;
      const float* d = side ? dscore + N : dscore;
      const int hi = seg_ptr[s + 1];
#pragma unroll 4
      for (int k = seg_ptr[s] + w; k < hi; k += 8) {
        const int i = seg_order[k];
        const float a = d[i];
        const float4 v = ld4(xc + (int64_t)i * ldx);
        acc.x = fmaf(a, v.x, acc.x);
        acc.y = fmaf(a, v.y, acc.y);
        acc.z = fmaf(a, v.z, acc.z);
        acc.w = fmaf(a, v.w, acc.w);
      }
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
    const float gs = (float)*gscale;
    st4(dH + g * 4 * C4 + 4 * c4, make_float4(t.x * gs, t.y * gs, t.z * gs, t.w * gs));
  }
}

// Node pass: gx_i = gscale (dpos_i H[b_i] + dneg_i H[(b_i + 1) mod G]) + dS[b_i] * S[b_i] * (1 - S[b_i]) / n_{b_i}: the two
// score paths and the pool path (sigmoid' then mean') in one write.  One thread per (row, float4 column).  A graph id outside
// [0, G) gets a zero row.
__global__ void __launch_bounds__(256)
k_infomax_node_bwd(int64_t N, int C4, const int64_t* __restrict__ batch, const int* __restrict__ seg_ptr, int64_t G,
                   const float* __restrict__ S, const float* __restrict__ H, const float* __restrict__ dS, const float* __restrict__ dscore,
                   const double* __restrict__ gscale, float* __restrict__ gx, int64_t ldgx) {
  pdl_prologue();
  const float gs = (float)*gscale;
  const int64_t total = N * C4;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / C4;
    const int c = (int)(idx - i * C4) * 4;
    const int64_t g = batch[i];
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g >= 0 && g < G) {
      const int64_t gn = g + 1 == G ? 0 : g + 1;
      const float a = __fmul_rn(dscore[i], gs), b = __fmul_rn(dscore[N + i], gs);
      const float inv = 1.f / (float)max(seg_ptr[g + 1] - seg_ptr[g], 1);
      const int64_t o = g * 4 * C4 + c;
      const float4 hp = ld4(H + o), hn = ld4(H + gn * 4 * C4 + c), s = ld4(S + o), d = ld4(dS + o);
      r.x = fmaf(b, hn.x, a * hp.x) + d.x * (s.x * (1.f - s.x)) * inv;
      r.y = fmaf(b, hn.y, a * hp.y) + d.y * (s.y * (1.f - s.y)) * inv;
      r.z = fmaf(b, hn.z, a * hp.z) + d.z * (s.z * (1.f - s.z)) * inv;
      r.w = fmaf(b, hn.w, a * hp.w) + d.w * (s.w * (1.f - s.w)) * inv;
    }
    st4(gx + i * ldgx + c, r);
  }
}

inline int64_t gc_bytes(int64_t G, int64_t C) { return align_up(G * C * (int64_t)sizeof(float), 256); }

}  // namespace

extern "C" {

int pgnn_infomax_summary_fwd(const float* x, int64_t ldx, const int32_t* seg_ptr, const int32_t* seg_order, int64_t G, int64_t C,
                             float* S, int64_t lds, void* stream) {
  PGNN_CHECK_ARG(G >= 0 && C > 0 && ldx >= C && lds >= C);
  if (G == 0) return PGNN_OK;
  PGNN_CHECK_ARG(seg_ptr && S);
  if (C % 4 || ldx % 4 || lds % 4 || !aligned16(x) || !aligned16(S)) return PGNN_EUNSUPPORTED;
  const int C4 = (int)(C / 4);
  PGNN_CUDA(pgnn_launch(k_infomax_summary_fwd, dim3((unsigned)G, (unsigned)ceil_div(C4, 32)), dim3(256), 0, as_stream(stream), x, ldx,
                        seg_ptr, seg_order, C4, S, lds));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int64_t pgnn_infomax_bce_workspace_bytes(void) { return (int64_t)sizeof(InfomaxBceWs); }

int pgnn_infomax_bce_fwd(const float* x, int64_t ldx, int64_t N, int64_t C, const int64_t* batch, const float* H, int64_t G,
                         double* loss, float* pos, float* neg, float* dscore, void* workspace, int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(N >= 0 && C > 0 && ldx >= C && G >= 0 && loss && workspace);
  PGNN_CHECK_ARG(N == 0 || (x && batch && H && G > 0 && pos && neg && dscore));
  if (workspace_bytes < (int64_t)sizeof(InfomaxBceWs)) return PGNN_EWORKSPACE;
  if (C % 4 || ldx % 4 || (x && !aligned16(x)) || (H && !aligned16(H))) return PGNN_EUNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  InfomaxBceWs* ws = reinterpret_cast<InfomaxBceWs*>(workspace);
  PGNN_CUDA(cudaMemsetAsync(&ws->ticket, 0, sizeof(unsigned int), st));
  int64_t blocks = ceil_div(N, (int64_t)kImxNodesPerCta);
  if (blocks > kImxMaxBlocks) blocks = kImxMaxBlocks;
  if (blocks < 1) blocks = 1;   // one CTA writes the loss of an empty batch (NaN)
  PGNN_CUDA(pgnn_launch(k_infomax_bce_fwd, dim3((unsigned)blocks), dim3(kImxThreads), 0, st, x, ldx, N, (int)(C / 4), batch, G, H, ws, loss,
                        pos, neg, dscore));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int64_t pgnn_infomax_bce_bwd_workspace_bytes(int64_t G, int64_t C) {
  if (G < 0 || C <= 0) return PGNN_EINVAL;
  return 2 * gc_bytes(G, C) + align_up(pgnn_tc_wgrad_workspace_floats(G, C, C) * (int64_t)sizeof(float), 256);
}

int pgnn_infomax_bce_bwd(const float* x, int64_t ldx, int64_t N, int64_t C, const int64_t* batch, const int32_t* seg_ptr,
                         const int32_t* seg_order, int64_t G, const float* S, const float* H, const float* W, const float* dscore,
                         const double* gscale, float* gx, int64_t ldgx, float* gW, int precision, void* workspace,
                         int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(N >= 0 && C > 0 && ldx >= C && G >= 0 && (gx == nullptr || ldgx >= C));
  PGNN_CHECK_ARG(N == 0 || G > 0);
  if (G == 0) return gW ? pgnn_linear_bwd_w(nullptr, C, nullptr, C, 0, C, C, gW, nullptr, precision, stream) : PGNN_OK;
  PGNN_CHECK_ARG(seg_ptr && S && H && W && gscale && workspace && (N == 0 || (x && batch && seg_order && dscore)));
  if (workspace_bytes < pgnn_infomax_bce_bwd_workspace_bytes(G, C)) return PGNN_EWORKSPACE;
  if (C % 4 || ldx % 4 || (gx && ldgx % 4) || (x && !aligned16(x)) || (gx && !aligned16(gx)) || !aligned16(S) || !aligned16(H) ||
      !aligned16(workspace))
    return PGNN_EUNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  const int C4 = (int)(C / 4);
  float* dH = reinterpret_cast<float*>(workspace);
  float* dS = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + gc_bytes(G, C));
  float* part = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 2 * gc_bytes(G, C));
  PGNN_CUDA(pgnn_launch(k_infomax_graph_reduce, dim3((unsigned)G, (unsigned)ceil_div(C4, 32)), dim3(256), 0, st, x, ldx, N, C4, seg_ptr,
                        seg_order, G, dscore, gscale, dH));
  PGNN_LAUNCH_CHECK();
  int rc;
  if (gW) {   // dW = S^T dH
    rc = precision == 1 ? pgnn_tc_linear_bwd_w_ws(S, C, dH, C, G, C, C, gW, nullptr, part, pgnn_tc_wgrad_workspace_floats(G, C, C), st)
                        : PGNN_EUNSUPPORTED;
    if (rc == PGNN_EUNSUPPORTED) rc = pgnn_linear_bwd_w(S, C, dH, C, G, C, C, gW, nullptr, precision, stream);
    if (rc != PGNN_OK) return rc;
  }
  if (gx == nullptr || N == 0) return PGNN_OK;
  if ((rc = pgnn_linear_fwd(dH, C, W, nullptr, G, C, C, 0, dS, C, precision, stream)) != PGNN_OK) return rc;         // dS = dH W^T
  PGNN_CUDA(pgnn_launch(k_infomax_node_bwd, dim3(grid_items(N * C4, 256)), dim3(256), 0, st, N, C4, batch, seg_ptr, G, S, H, dS, dscore,
                        gscale, gx, ldgx));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

}  // extern "C"
