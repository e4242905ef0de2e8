// Whole-encoder entry points for the chem GNN with gnn_type = "gcn" | "graphsage" | "gat" (chem/model.py:58-202 conv
// layers inside GNN.forward :255-290, JK="last", drop_ratio=0): like pgnn_chem_gin_* (encoder.cu), ONE call enqueues the graph
// preparation, the atom embedding and all L x (Linear -> propagate [-> L2-normalise] -> BatchNorm [-> ReLU]) layers, a second
// call the whole backward, and the gradients leave in ONE flat fp32 buffer.  The per-layer arithmetic is the operator-level
// C ABI of include/pgnn_b200.h (the same kernels the layer-by-layer Python composition launches); what this file removes is
// the ~100 Python/ctypes crossings, the per-op allocations and the torch.cat of the two bond tables per layer and pass.
//
//   GCN        (chem/model.py:85-104):   xl = Linear(D,D)(h);  out_i = sum_j d_i^-1/2 d_j^-1/2 (xl_j + e_ij)
//   GraphSAGE  (chem/model.py:182-202):  xl = Linear(D,D)(h);  out_i = normalize(mean_j (xl_j + e_ij))
//   GAT        (chem/model.py:134-165):  xl = Linear(D,2D)(h); out_i = mean_heads(sum_j alpha_ij (xl_j + e_ij)) + bias
// each followed by BatchNorm1d(D) and, except after the last layer, ReLU (chem/model.py:267-276).
#include "common.cuh"

#include <cstdlib>
#include <map>
#include <mutex>

int pgnn_internal_edge_table_bwd2(const float* S, int Q, const float* g, int64_t ldg, int64_t g_off, int64_t n, int C, float* gT,
                                  int64_t ldt, float* gT2, int q_split, cudaStream_t st);
int pgnn_internal_aggregate_fwd(const float* x, int64_t ldx, const float* in_scale, const float* in_shift, int in_relu,
                                int64_t num_nodes, int64_t C, const int32_t* rowptr_t, const int32_t* nbr_t, int mode, const float* dinv,
                                const float* S, int64_t Q, const float* T, const float* T2, int q_split, int64_t edge_off, float* out,
                                int64_t ldo, cudaStream_t st, const PgnnBnFold* fold);
int pgnn_internal_chem_onehot(const int64_t* x, int64_t n, int rows1, int rows2, float* onehot, int64_t ld, cudaStream_t st);
int pgnn_tc_linear_bwd_w_ws(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t N, int64_t K, float* gw,
                            float* gb, float* partials, int64_t partial_floats, cudaStream_t st);
int64_t pgnn_tc_wgrad_workspace_floats(int64_t M, int64_t N, int64_t K);

namespace {

constexpr int kAtomRows = 120, kChiralRows = 3, kOneHotLd = 124;
constexpr int kHeads = 2;          // chem/model.py:108 (heads=2 is what GNN.__init__ builds, :243)
constexpr float kSlope = 0.2f;     // negative_slope, chem/model.py:108

enum { P_XEMB1 = 0, P_XEMB2 = 1, P_LAYER0 = 2 };
// per-layer parameter order (also the flat gradient order); the two bond tables are adjacent so that one [9, C] block holds both
enum { G_W = 0, G_B, G_ET1, G_ET2, G_GAMMA, G_BETA, G_COUNT };                    // gcn / graphsage
enum { A_W = 0, A_B, A_ATT, A_BIAS, A_ET1, A_ET2, A_GAMMA, A_BETA, A_COUNT };     // gat

inline int layer_params(int type) { return type == PGNN_CONV_GAT ? A_COUNT : G_COUNT; }
inline int agg_mode(int type) { return type == PGNN_CONV_GCN ? PGNN_AGG_GCN : PGNN_AGG_MEAN; }

struct Carve {
  char* base;
  int64_t off = 0;
  explicit Carve(void* b) : base(reinterpret_cast<char*>(b)) {}
  template <typename T>
  T* take(int64_t count) {
    T* p = reinterpret_cast<T*>(base + off);
    off += align_up((count > 0 ? count : 1) * (int64_t)sizeof(T), 256);
    return p;
  }
};

struct Ws {
  int32_t *rowptr_t, *rowptr_s, *nbr_t, *eid_t, *nbr_s, *eid_s;
  float *S, *dinv, *h0, *onehot;
  float *xl, *z, *hout;        // per layer: Linear output [N, HD], BatchNorm input [N, D], layer output [N, D]
  float *nrm, *alpha, *pq, *T; // per layer: SAGE row norms [N]; GAT attention [(E+N), H], logit halves [N, H, 2], tables [9, HD]
  float *mean, *invstd;        // [L, D]
  float *gz, *ga, *gxl, *gh;   // backward temporaries [N, D], [N, D], [N, HD], [N, D]
  float* wpart;
  int64_t wpart_floats;
  void* scratch;
  int64_t scratch_bytes, total;
};

Ws carve(void* base, int type, int64_t N, int64_t E, int64_t L, int64_t D) {
  Carve c(base);
  Ws w;
  const int64_t HD = type == PGNN_CONV_GAT ? kHeads * D : D;
  w.rowptr_t = c.take<int32_t>(N + 1);
  w.rowptr_s = c.take<int32_t>(N + 1);
  w.nbr_t = c.take<int32_t>(E);
  w.eid_t = c.take<int32_t>(E);
  w.nbr_s = c.take<int32_t>(E);
  w.eid_s = c.take<int32_t>(E);
  w.S = c.take<float>(N * 9);
  w.dinv = c.take<float>(N);
  w.h0 = c.take<float>(N * D);
  w.onehot = c.take<float>(N * kOneHotLd);
  w.xl = c.take<float>(L * N * HD);
  w.z = c.take<float>(L * N * D);
  w.hout = c.take<float>(L * N * D);
  w.nrm = c.take<float>(type == PGNN_CONV_SAGE ? L * N : 0);
  w.alpha = c.take<float>(type == PGNN_CONV_GAT ? L * (E + N) * kHeads : 0);
  w.pq = c.take<float>(type == PGNN_CONV_GAT ? L * N * kHeads * 2 : 0);
  w.T = c.take<float>(type == PGNN_CONV_GAT ? L * 9 * HD : 0);
  w.mean = c.take<float>(L * D);
  w.invstd = c.take<float>(L * D);
  w.gz = c.take<float>(N * D);
  w.ga = c.take<float>(N * D);
  w.gxl = c.take<float>(2 * N * HD);   // two copies by layer parity: the side-stream wgrad of layer l reads one while layer l-1 writes the other
  w.gh = c.take<float>(N * D);
  w.wpart_floats = pgnn_tc_wgrad_workspace_floats(N, HD, D);
  {
    const int64_t e = pgnn_tc_wgrad_workspace_floats(N, kAtomRows + kChiralRows, D);  // the embedding tables' gradient as a GEMM
    if (e > w.wpart_floats) w.wpart_floats = e;
  }
  w.wpart = c.take<float>(w.wpart_floats);
  int64_t sb = pgnn_graph_prep_workspace_bytes(N, E);
  const int64_t bb = pgnn_bn_workspace_bytes(N > 0 ? N : 1, D);
  if (bb > sb) sb = bb;
  if (type == PGNN_CONV_GAT) {
    const int64_t gb = pgnn_gat_bwd_workspace_bytes(N, E, kHeads, D);
    if (gb > sb) sb = gb;
  }
  w.scratch_bytes = sb;
  w.scratch = c.take<char>(sb);
  w.total = c.off;
  return w;
}

// weight-gradient GEMMs on a side stream, as in encoder.cu: they only feed the gradient buffer, so they run under the next
// layer's BatchNorm / attention / gather kernels instead of in front of them.  PGNN_WGRAD_STREAM=0 disables.
struct SideCtx {
  cudaStream_t side = nullptr;
  cudaEvent_t gxl_ready[2] = {}, w_done[2] = {}, join = nullptr;
  bool ok = false;
};
SideCtx* side_ctx(cudaStream_t main_stream) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, SideCtx*> all;
  static int enabled = -1;
  std::lock_guard<std::mutex> g(mu);
  if (enabled < 0) {
    const char* e = getenv("PGNN_WGRAD_STREAM");
    enabled = (e && e[0] == '0') ? 0 : 1;
  }
  // the per-kernel timing mode (pgnn_profile_enable) wants each kernel's own duration: no concurrent stream while it is on
  if (!enabled || g_pgnn_profile_on.load(std::memory_order_relaxed) != 0) return nullptr;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  auto key = std::make_pair(dev, main_stream);
  auto it = all.find(key);
  if (it != all.end()) return it->second->ok ? it->second : nullptr;
  SideCtx* c = new SideCtx();
  all[key] = c;
  bool ok = cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking) == cudaSuccess;
  for (int i = 0; i < 2 && ok; ++i)
    ok = cudaEventCreateWithFlags(&c->gxl_ready[i], cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&c->w_done[i], cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&c->join, cudaEventDisableTiming) == cudaSuccess;
  if (!ok) cudaGetLastError();
  c->ok = ok;
  return ok ? c : nullptr;
}

bool valid_type(int t) { return t == PGNN_CONV_GCN || t == PGNN_CONV_SAGE || t == PGNN_CONV_GAT; }

// PGNN_EMBED_GEMM=0: embedding-table gradient through the vector-atomics kernel instead of the one-hot GEMM (development switch)
inline bool embed_gemm_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("PGNN_EMBED_GEMM");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

#define TRY(call)                     \
  do {                                \
    int rc__ = (call);                \
    if (rc__ != PGNN_OK) return rc__; \
  } while (0)

}  // namespace

extern "C" {

int64_t pgnn_chem_conv_num_params(int conv_type, int64_t L) {
  if (!valid_type(conv_type) || L < 1) return PGNN_EINVAL;
  return 2 + (int64_t)layer_params(conv_type) * L;
}

int pgnn_chem_conv_grad_offsets(int conv_type, int64_t L, int64_t D, int64_t* offsets) {
  PGNN_CHECK_ARG(valid_type(conv_type) && L >= 1 && D > 0 && offsets);
  const int64_t HD = conv_type == PGNN_CONV_GAT ? kHeads * D : D;
  int64_t o = 0, i = 0;
  offsets[i++] = o; o += kAtomRows * D;
  offsets[i++] = o; o += kChiralRows * D;
  for (int64_t l = 0; l < L; ++l) {
    offsets[i++] = o; o += HD * D;   // linear.weight / weight_linear.weight [HD, D]
    offsets[i++] = o; o += HD;       // its bias
    if (conv_type == PGNN_CONV_GAT) {
      offsets[i++] = o; o += kHeads * 2 * D;  // att [1, H, 2D]
      offsets[i++] = o; o += D;               // bias [D]
    }
    offsets[i++] = o; o += 6 * HD;   // edge_embedding1.weight
    offsets[i++] = o; o += 3 * HD;   // edge_embedding2.weight
    offsets[i++] = o; o += D;        // batch_norms.l.weight
    offsets[i++] = o; o += D;        // batch_norms.l.bias
  }
  offsets[i] = o;
  return PGNN_OK;
}

int64_t pgnn_chem_conv_workspace_bytes(int conv_type, int64_t N, int64_t E, int64_t L, int64_t D) {
  if (!valid_type(conv_type) || N < 0 || E < 0 || L < 1 || D <= 0) return PGNN_EINVAL;
  return carve(nullptr, conv_type, N, E, L, D).total;
}

int pgnn_chem_conv_forward(int conv_type, const void* const* params, void* const* bn_running_mean, void* const* bn_running_var,
                           void* const* bn_num_batches_tracked, const int64_t* x, const int64_t* edge_index, const int64_t* edge_attr,
                           int64_t N, int64_t E, int64_t L, int64_t D, int training, float momentum, float eps, int precision,
                           float* node_rep, int64_t ld_out, void* workspace, int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(valid_type(conv_type) && N >= 0 && E >= 0 && L >= 1 && D > 0 && D % 4 == 0 && params && bn_running_mean && bn_running_var &&
                 workspace);
  PGNN_CHECK_ARG(N == 0 || (x && node_rep));
  PGNN_CHECK_ARG(E == 0 || (edge_index && edge_attr));
  if (workspace_bytes < pgnn_chem_conv_workspace_bytes(conv_type, N, E, L, D)) return PGNN_EWORKSPACE;
  if (N == 0) return PGNN_OK;
  cudaStream_t st = as_stream(stream);
  const bool gat = conv_type == PGNN_CONV_GAT;
  const int64_t HD = gat ? kHeads * D : D;
  const int PL = layer_params(conv_type);
  Ws w = carve(workspace, conv_type, N, E, L, D);
  TRY(pgnn_graph_prep(edge_index, E, N, w.rowptr_t, w.nbr_t, w.eid_t, w.rowptr_s, w.nbr_s, w.eid_s, w.scratch, w.scratch_bytes, stream));
  if (conv_type == PGNN_CONV_GCN) TRY(pgnn_gcn_dinv(w.rowptr_t, N, w.dinv, stream));
  if (!gat) TRY(pgnn_chem_edge_summary(edge_attr, w.rowptr_t, w.nbr_t, w.eid_t, N, agg_mode(conv_type), w.dinv, w.S, stream));
  TRY(pgnn_chem_embed_fwd(x, (const float*)params[P_XEMB1], kAtomRows, (const float*)params[P_XEMB2], kChiralRows, N, D, w.h0, D, stream));
  if (training && precision == 1) TRY(pgnn_internal_chem_onehot(x, N, kAtomRows, kChiralRows, w.onehot, kOneHotLd, st));
  const float* h = w.h0;
  for (int64_t l = 0; l < L; ++l) {
    const void* const* p = params + P_LAYER0 + l * PL;
    const bool last = l == L - 1;
    float* xl = w.xl + l * N * HD;
    float* z = w.z + l * N * D;
    float* hout = last ? node_rep : w.hout + l * N * D;
    const int64_t ldh = last ? ld_out : D;
    TRY(pgnn_linear_fwd(h, D, (const float*)p[gat ? A_W : G_W], (const float*)p[gat ? A_B : G_B], N, HD, D, 0, xl, HD, precision, stream));
    if (gat) {
      float* T = w.T + l * 9 * HD;  // the kernels index one [9, H*D] table: rows 0..5 bond type, 6..8 bond direction
      PGNN_CUDA(cudaMemcpyAsync(T, p[A_ET1], sizeof(float) * 6 * HD, cudaMemcpyDeviceToDevice, st));
      PGNN_CUDA(cudaMemcpyAsync(T + 6 * HD, p[A_ET2], sizeof(float) * 3 * HD, cudaMemcpyDeviceToDevice, st));
      TRY(pgnn_gat_fwd(xl, N, kHeads, D, (const float*)p[A_ATT], T, 0, edge_attr, w.rowptr_t, w.nbr_t, w.eid_t, E, (const float*)p[A_BIAS], kSlope,
                       w.alpha + l * (E + N) * kHeads, w.pq + l * N * kHeads * 2, z, D, stream));
    } else if (conv_type == PGNN_CONV_GCN) {
      TRY(pgnn_internal_aggregate_fwd(xl, D, nullptr, nullptr, 0, N, D, w.rowptr_t, w.nbr_t, PGNN_AGG_GCN, w.dinv, w.S, 9, (const float*)p[G_ET1],
                                      (const float*)p[G_ET2], 6, 0, z, D, st, nullptr));
    } else {
      // mean aggregation into the backward scratch `gz` (only its normalised rows and their norms are needed later)
      TRY(pgnn_internal_aggregate_fwd(xl, D, nullptr, nullptr, 0, N, D, w.rowptr_t, w.nbr_t, PGNN_AGG_MEAN, nullptr, w.S, 9, (const float*)p[G_ET1],
                                      (const float*)p[G_ET2], 6, 0, w.gz, D, st, nullptr));
      TRY(pgnn_l2norm_fwd(w.gz, D, N, D, z, D, w.nrm + l * N, stream));
    }
    const float* gamma = (const float*)p[gat ? A_GAMMA : G_GAMMA];
    const float* beta = (const float*)p[gat ? A_BETA : G_BETA];
    if (training) {
      TRY(pgnn_bn_fwd_train(z, D, N, D, gamma, beta, (float*)bn_running_mean[l], (float*)bn_running_var[l],
                            bn_num_batches_tracked ? (int64_t*)bn_num_batches_tracked[l] : nullptr, momentum, eps, !last, hout, ldh, w.mean + l * D,
                            w.invstd + l * D, nullptr, nullptr, w.scratch, w.scratch_bytes, stream));
    } else {
      TRY(pgnn_bn_fwd_eval(z, D, N, D, gamma, beta, (const float*)bn_running_mean[l], (const float*)bn_running_var[l], eps, !last, hout, ldh, stream));
    }
    h = hout;
  }
  return PGNN_OK;
}

int pgnn_chem_conv_backward(int conv_type, const void* const* params, const float* g_node_rep, int64_t ldg, const int64_t* x,
                            const int64_t* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D, int precision, float* grads,
                            void* workspace, int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(valid_type(conv_type) && N >= 0 && E >= 0 && L >= 1 && L <= 64 && D > 0 && D % 4 == 0 && params && grads && workspace);
  if (workspace_bytes < pgnn_chem_conv_workspace_bytes(conv_type, N, E, L, D)) return PGNN_EWORKSPACE;
  int64_t off[2 + A_COUNT * 64 + 1];
  pgnn_chem_conv_grad_offsets(conv_type, L, D, off);
  cudaStream_t st = as_stream(stream);
  const bool gat = conv_type == PGNN_CONV_GAT;
  const int64_t HD = gat ? kHeads * D : D;
  const int PL = layer_params(conv_type);
  if (N == 0) {
    PGNN_CUDA(cudaMemsetAsync(grads, 0, sizeof(float) * off[2 + PL * L], st));
    return PGNN_OK;
  }
  PGNN_CHECK_ARG(g_node_rep && x && (E == 0 || edge_attr));
  Ws w = carve(workspace, conv_type, N, E, L, D);
  const float* gy = g_node_rep;
  int64_t ldgy = ldg;
  SideCtx* sc = precision == 1 ? side_ctx(st) : nullptr;
  cudaStream_t wst = sc ? sc->side : st;
  for (int64_t l = L - 1; l >= 0; --l) {
    const void* const* p = params + P_LAYER0 + l * PL;
    const int64_t* o = off + P_LAYER0 + l * PL;
    const bool last = l == L - 1;
    const int par = (int)(l & 1);
    const float* xl = w.xl + l * N * HD;
    const float* z = w.z + l * N * D;
    const float* hin = l == 0 ? w.h0 : w.hout + (l - 1) * N * D;
    float* gxl = w.gxl + (sc ? par * N * HD : 0);
    const float* gamma = (const float*)p[gat ? A_GAMMA : G_GAMMA];
    const float* beta = (const float*)p[gat ? A_BETA : G_BETA];
    TRY(pgnn_bn_bwd(gy, ldgy, z, D, N, D, gamma, beta, w.mean + l * D, w.invstd + l * D, !last, w.gz, D, grads + o[gat ? A_GAMMA : G_GAMMA],
                    grads + o[gat ? A_BETA : G_BETA], w.scratch, w.scratch_bytes, stream));
    if (sc) PGNN_CUDA(cudaStreamWaitEvent(st, sc->w_done[par], 0));  // layer l+2's wgrad has finished reading this copy of gxl
    if (gat) {
      // gT [9, HD] lands on the two adjacent bond-table gradients
      TRY(pgnn_gat_bwd(w.gz, D, xl, N, kHeads, D, (const float*)p[A_ATT], w.T + l * 9 * HD, 0, edge_attr, w.rowptr_t, w.nbr_t, w.eid_t, w.rowptr_s,
                       w.nbr_s, w.eid_s, E, kSlope, w.alpha + l * (E + N) * kHeads, w.pq + l * N * kHeads * 2, gxl, grads + o[A_ATT],
                       grads + o[A_ET1], grads + o[A_BIAS], w.scratch, w.scratch_bytes, stream));
    } else {
      const float* ga = w.gz;
      if (conv_type == PGNN_CONV_SAGE) {
        TRY(pgnn_l2norm_bwd(w.gz, D, z, D, w.nrm + l * N, N, D, w.ga, D, stream));
        ga = w.ga;
      }
      PGNN_CUDA(cudaMemsetAsync(grads + o[G_ET1], 0, sizeof(float) * 9 * D, st));
      TRY(pgnn_internal_edge_table_bwd2(w.S, 9, ga, D, 0, N, (int)D, grads + o[G_ET1], D, grads + o[G_ET2], 6, st));
      TRY(pgnn_aggregate_bwd(ga, D, N, D, w.rowptr_s, w.nbr_s, agg_mode(conv_type), w.dinv, w.rowptr_t, gxl, D, stream));
    }
    // Linear backward: weight + bias gradients (side stream), then the input gradient
    if (sc) {
      PGNN_CUDA(cudaEventRecord(sc->gxl_ready[par], st));
      PGNN_CUDA(cudaStreamWaitEvent(wst, sc->gxl_ready[par], 0));
    }
    int rc = PGNN_EUNSUPPORTED;
    if (precision == 1)
      rc = pgnn_tc_linear_bwd_w_ws(gxl, HD, hin, D, N, HD, D, grads + o[gat ? A_W : G_W], grads + o[gat ? A_B : G_B], w.wpart, w.wpart_floats, wst);
    if (rc == PGNN_EUNSUPPORTED) {
      if (sc) {
        PGNN_CUDA(cudaEventRecord(sc->join, wst));
        PGNN_CUDA(cudaStreamWaitEvent(st, sc->join, 0));
      }
      rc = pgnn_linear_bwd_w(gxl, HD, hin, D, N, HD, D, grads + o[gat ? A_W : G_W], grads + o[gat ? A_B : G_B], precision, stream);
    } else if (sc) {
      PGNN_CUDA(cudaEventRecord(sc->w_done[par], wst));
    }
    if (rc != PGNN_OK) return rc;
    TRY(pgnn_linear_bwd_x(gxl, HD, (const float*)p[gat ? A_W : G_W], N, HD, D, nullptr, 0, w.gh, D, precision, stream));
    gy = w.gh;
    ldgy = D;
  }
  if (sc) {  // the side stream's last wgrad (and its use of the split-K workspace) before the embedding GEMM and before returning
    PGNN_CUDA(cudaEventRecord(sc->join, wst));
    PGNN_CUDA(cudaStreamWaitEvent(st, sc->join, 0));
  }
  int rc_e = PGNN_EUNSUPPORTED;
  if (precision == 1 && embed_gemm_enabled())
    rc_e = pgnn_tc_linear_bwd_w_ws(w.onehot, kOneHotLd, w.gh, D, N, kAtomRows + kChiralRows, D, grads + off[P_XEMB1], nullptr, w.wpart, w.wpart_floats, st);
  if (rc_e == PGNN_EUNSUPPORTED)
    rc_e = pgnn_chem_embed_bwd(x, w.gh, D, N, D, grads + off[P_XEMB1], kAtomRows, grads + off[P_XEMB2], kChiralRows, stream);
  return rc_e;
}

}  // extern "C"
