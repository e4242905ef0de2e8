// Whole-encoder entry points for the chem GNN (chem/model.py:206-290 with JK="last", any drop_ratio): ONE call enqueues graph
// preparation, the atom embedding and all L layers; a second call enqueues the whole backward.  This is what GNN.forward binds
// to, so a training step crosses the Python/C boundary twice instead of ~60 (GIN) or ~100 (conv types) times, without the
// per-op allocations and the torch.cat of the two bond tables per layer and pass.
//
//   GIN        (pgnn_chem_gin_*, chem/model.py:37-55):  L x (aggregate -> MLP -> BatchNorm[-> ReLU]).  The inter-layer
//              BatchNorm + ReLU never makes a pass of its own: layer l only accumulates the batch statistics and layer l+1's
//              gather applies scale/shift/ReLU while it loads the rows (pgnn_aggregate_fwd's in_scale/in_shift).
//   pgnn_chem_conv_* with conv_type =
//   GCN        (chem/model.py:85-104):   xl = Linear(D,D)(h);  out_i = sum_j d_i^-1/2 d_j^-1/2 (xl_j + e_ij)
//   GraphSAGE  (chem/model.py:182-202):  xl = Linear(D,D)(h);  out_i = normalize(mean_j (xl_j + e_ij))
//   GAT        (chem/model.py:134-165):  xl = Linear(D,2D)(h); out_i = mean_heads(sum_j alpha_ij (xl_j + e_ij)) + bias
//   each followed by BatchNorm1d(D) and, except after the last layer, ReLU (chem/model.py:267-276).  The per-layer arithmetic
//   is the operator-level C ABI of include/pgnn_b200.h (the same kernels the layer-by-layer Python composition launches).
//
// Dropout (training, drop_p > 0; chem/model.py:271-275) never makes a pass of its own either: layer l's mask (PgnnDropout with
// layer = l, common.cuh) is applied by whichever kernel materialises or loads layer l's output -- GIN: the next layer's gather
// and, for the last layer, the BatchNorm apply that writes node_rep; the conv types: the BatchNorm apply that writes hout.  The
// backward applies it to the incoming gradient inside the BatchNorm backward.  drop_p == 0 launches exactly the kernels without
// a mask.
//
// Parameters arrive as a host array of device pointers in a fixed order, gradients leave in ONE flat fp32 buffer with the
// library-defined layout of pgnn_chem_gin_grad_offsets / pgnn_chem_conv_grad_offsets (grad_layout below), which is also the
// buffer the data-parallel all-reduce runs on.
//
// The bio GNN (bio/model.py, pgnn_bio_encoder_*) runs on the same scaffolding: workspace carving (Carve / Front / Tail), Drops,
// the side-stream weight gradients (side_wgrad) and a flat gradient layout.  Its GIN has a layer body of its own (bio_gin_*);
// GCN / GraphSAGE / GAT share one body with chem (conv_forward / conv_backward), the domain filling in the layer's edge term
// (EdgeTerm) and the step around the conv: chem's BatchNorm, bio's ReLU + dropout sweep.
#include "common.cuh"

#include <cstdlib>
#include <map>
#include <mutex>
#include <vector>

int pgnn_internal_edge_table_bwd2(const float* S, int Q, const float* g, int64_t ldg, int64_t g_off, int64_t n, int C, float* gT,
                                  int64_t ldt, float* gT2, int q_split, cudaStream_t st);
int pgnn_internal_aggregate_fwd(const float* x, int64_t ldx, const float* in_scale, const float* in_shift, int in_relu,
                                int64_t num_nodes, int64_t C, const int32_t* rowptr_t, const int32_t* nbr_t, int mode, const float* dinv,
                                const float* S, int64_t Q, const float* T, const float* T2, int q_split, int64_t edge_off, float* out,
                                int64_t ldo, cudaStream_t st, const PgnnBnFold* fold, const PgnnDropout* drop);

int pgnn_internal_chem_onehot(const int64_t* x, int64_t n, int rows1, int rows2, float* onehot, int64_t ld, cudaStream_t st);

int pgnn_tc_linear_fwd(const float*, int64_t, const float*, const float*, int64_t, int64_t, int64_t, int, float*, int64_t,
                       cudaStream_t, const PgnnGemmHooks*);
int pgnn_tc_linear_bwd_x(const float*, int64_t, const float*, int64_t, int64_t, int64_t, const float*, int64_t, float*, int64_t,
                         cudaStream_t, const PgnnGemmHooks*);
int pgnn_tc_linear_bwd_w_ws(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t N, int64_t K, float* gw,
                            float* gb, float* partials, int64_t partial_floats, cudaStream_t st);
int64_t pgnn_tc_wgrad_workspace_floats(int64_t M, int64_t N, int64_t K);
int64_t pgnn_tc_image_floats(int64_t rows, int64_t k);
int pgnn_internal_pack_images(int count, const float* const* w, const int64_t* ld, const int* rows, const int* cols, const int* trans,
                              float* const* img, cudaStream_t st);
int pgnn_tc_linear_fwd_img(const float* x, int64_t ldx, const float* img, int64_t img_r, int64_t img_k, const float* bias, int64_t M,
                           int64_t N, int64_t K, int relu, float* y, int64_t ldy, cudaStream_t st, const PgnnGemmHooks* hooks);
int pgnn_tc_linear_bwd_x_img(const float* gy, int64_t ldgy, const float* img, int64_t img_r, int64_t img_k, int64_t M, int64_t N,
                             int64_t K, const float* relu_src, int64_t ldr, float* gx, int64_t ldgx, cudaStream_t st,
                             const PgnnGemmHooks* hooks);
int pgnn_internal_bn_apply_fold(const float* x, int64_t ldx, int64_t M, int64_t C, const PgnnBnFold& fold, int relu, float* y,
                                int64_t ldy, cudaStream_t st, const PgnnDropout* drop);
int pgnn_internal_bn_fwd_train(const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma, const float* beta,
                               float* running_mean, float* running_var, int64_t* num_batches_tracked, float momentum, float eps,
                               int relu, float* y, int64_t ldy, float* save_mean, float* save_invstd, float* scale, float* shift,
                               void* workspace, int64_t workspace_bytes, void* stream, const PgnnDropout* drop);
int pgnn_internal_bn_bwd(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma,
                         const float* beta, const float* save_mean, const float* save_invstd, int relu, float* gx, int64_t ldgx,
                         float* ggamma, float* gbeta, float* colsum, void* workspace, int64_t workspace_bytes, cudaStream_t st,
                         const PgnnDropout* drop);

namespace {

constexpr int kGin = 0;            // GIN's type code inside this file; the conv types use PGNN_CONV_* (never 0)
constexpr int kAtomRows = 120, kChiralRows = 3;   // chem/model.py:9-10
constexpr int kOneHotLd = 124;                    // kAtomRows + kChiralRows padded to a multiple of 4
constexpr int kHeads = 2;          // chem/model.py:108 (heads=2 is what GNN.__init__ builds, :243)
constexpr float kSlope = 0.2f;     // negative_slope, chem/model.py:108
constexpr int kChemQ = 9, kChemQSplit = 6;  // chem S columns: 6 bond-type rows (edge_embedding1), then 3 direction rows
constexpr int kBioQ = 10;          // bio S columns: the 9 edge attributes + the weight sum that multiplies the encoder bias

// order of the parameter pointer table and of the flat gradient layout
enum { P_XEMB1 = 0, P_XEMB2 = 1, P_LAYER0 = 2 };
// per-layer parameter order; the two bond tables are adjacent so that one [9, C] block holds both
enum { L_W1 = 0, L_B1, L_W2, L_B2, L_ET1, L_ET2, L_GAMMA, L_BETA, L_COUNT };     // gin
enum { G_W = 0, G_B, G_ET1, G_ET2, G_GAMMA, G_BETA, G_COUNT };                    // gcn / graphsage
enum { A_W = 0, A_B, A_ATT, A_BIAS, A_ET1, A_ET2, A_GAMMA, A_BETA, A_COUNT };     // gat
// the leading parameters of a conv layer, the same in both domains (BioParam below): the Linear, then GAT's att and bias
constexpr int CV_W = 0, CV_B = 1, CV_ATT = 2, CV_BIAS = 3;
static_assert(G_W == CV_W && G_B == CV_B && A_W == CV_W && A_B == CV_B && A_ATT == CV_ATT && A_BIAS == CV_BIAS, "chem conv order");

inline int layer_params(int type) { return type == kGin ? L_COUNT : type == PGNN_CONV_GAT ? A_COUNT : G_COUNT; }
inline int agg_mode(int type) { return type == kGin ? PGNN_AGG_SUM : type == PGNN_CONV_GCN ? PGNN_AGG_GCN : PGNN_AGG_MEAN; }
bool valid_conv(int t) { return t == PGNN_CONV_GCN || t == PGNN_CONV_SAGE || t == PGNN_CONV_GAT; }
bool valid_type(int t) { return t == kGin || valid_conv(t); }

// Per-layer dropout of one pass: layer l's mask is PgnnDropout(p, seed, l).  p == 0 (or eval mode) leaves every layer without
// one, so the kernels without a mask run.
struct Drops {
  float p = 0.f;
  int64_t seed = 0;
  PgnnDropout at(int64_t l) const {
    PgnnDropout d;
    pgnn_make_dropout(p, seed, l, &d);
    return d;
  }
};

// The BatchNorm running state of a pass (one pointer per layer; nbt may be null) and its hyper-parameters
struct BnRun {
  void* const* mean = nullptr;
  void* const* var = nullptr;
  void* const* nbt = nullptr;
  float momentum = 0.f, eps = 0.f;
  float* rm(int64_t l) const { return (float*)mean[l]; }
  float* rv(int64_t l) const { return (float*)var[l]; }
  int64_t* nb(int64_t l) const { return nbt ? (int64_t*)nbt[l] : nullptr; }
};

#define TRY(call)                     \
  do {                                \
    int rc__ = (call);                \
    if (rc__ != PGNN_OK) return rc__; \
  } while (0)

// The flat gradient layout of one type: fills offsets[0..count] when given and returns the parameter count.
int64_t grad_layout(int type, int64_t L, int64_t D, int64_t* offsets) {
  if (!offsets) return 2 + (int64_t)layer_params(type) * L;
  const int64_t HD = type == PGNN_CONV_GAT ? kHeads * D : D;
  int64_t o = 0, i = 0;
  auto next = [&](int64_t size) { offsets[i++] = o; o += size; };
  next(kAtomRows * D);    // x_embedding1.weight
  next(kChiralRows * D);  // x_embedding2.weight
  for (int64_t l = 0; l < L; ++l) {
    if (type == kGin) {
      next(2 * D * D);  // mlp.0.weight [2D, D]
      next(2 * D);      // mlp.0.bias
      next(2 * D * D);  // mlp.2.weight [D, 2D]
      next(D);          // mlp.2.bias
    } else {
      next(HD * D);     // linear.weight / weight_linear.weight [HD, D]
      next(HD);         // its bias
      if (type == PGNN_CONV_GAT) {
        next(kHeads * 2 * D);  // att [1, H, 2D]
        next(D);               // bias [D]
      }
    }
    next(6 * HD);  // edge_embedding1.weight
    next(3 * HD);  // edge_embedding2.weight
    next(D);       // batch_norms.l.weight
    next(D);       // batch_norms.l.bias
  }
  offsets[i] = o;
  return i;
}

// 256-byte aligned regions of one workspace (base == nullptr only measures); an empty region takes no space
struct Carve {
  char* base;
  int64_t off = 0;
  explicit Carve(void* b) : base(reinterpret_cast<char*>(b)) {}
  template <typename T>
  T* take(int64_t count) {
    T* p = reinterpret_cast<T*>(base + off);
    off += align_up(count * (int64_t)sizeof(T), 256);
    return p;
  }
};

// the first regions of every workspace: what the prologues write
struct Front {
  int32_t *rowptr_t, *rowptr_s, *nbr_t, *eid_t, *nbr_s, *eid_s;
  float *S, *dinv, *h0;  // dinv: conv types only
  float* onehot;         // chem: [N, kOneHotLd] atom-code one-hot rows (embedding gradient as a GEMM)
};

void carve_front(Carve& c, Front& f, bool bio, int type, int64_t N, int64_t E, int64_t D) {
  const int64_t e1 = E > 0 ? E : 1;
  f.rowptr_t = c.take<int32_t>(N + 1);
  f.rowptr_s = c.take<int32_t>(N + 1);
  f.nbr_t = c.take<int32_t>(e1);
  f.eid_t = c.take<int32_t>(e1);
  f.nbr_s = c.take<int32_t>(e1);
  f.eid_s = c.take<int32_t>(e1);
  f.S = c.take<float>(N * (bio ? kBioQ : kChemQ));
  f.dinv = type == kGin ? nullptr : c.take<float>(N);
  f.h0 = c.take<float>(N * D);
  f.onehot = bio ? nullptr : c.take<float>(N * kOneHotLd);
}

// the last regions of every workspace: split-K partial tiles of the largest weight-gradient GEMM, and one scratch shared by graph
// preparation, the BatchNorms (bn_width: the widest one; 0: none) and the GAT backward
struct Tail {
  float* wpart;
  int64_t wpart_floats;
  void* scratch;
  int64_t scratch_bytes, total;
};

void carve_tail(Carve& c, Tail& t, int type, int64_t N, int64_t E, int64_t D, int64_t wpart_floats, int64_t bn_width) {
  t.wpart_floats = wpart_floats;
  t.wpart = c.take<float>(wpart_floats);
  int64_t sb = pgnn_graph_prep_workspace_bytes(N, E);
  const int64_t bb = bn_width ? pgnn_bn_workspace_bytes(N > 0 ? N : 1, bn_width) : 0;
  const int64_t gb = type == PGNN_CONV_GAT ? pgnn_gat_bwd_workspace_bytes(N, E, kHeads, D) : 0;
  if (bb > sb) sb = bb;
  if (gb > sb) sb = gb;
  t.scratch_bytes = sb;
  t.scratch = c.take<char>(sb);
  t.total = c.off;
}

// chem split-K partial tiles: the layer wgrads ([width, D] over N rows) and the embedding tables' gradient as a GEMM
int64_t split_k_floats(int64_t N, int64_t width, int64_t D) {
  const int64_t a = pgnn_tc_wgrad_workspace_floats(N, width, D);
  const int64_t e = pgnn_tc_wgrad_workspace_floats(N, kAtomRows + kChiralRows, D);
  return e > a ? e : a;
}

struct GinWs : Front, Tail {
  float *scale, *shift, *mean, *invstd;  // [L, D]
  double* bn_acc;                        // [L][2][D] fp64 BatchNorm sums of the forward
  float *aggr, *z1, *z2;                 // [L, N, D], [L, N, 2D], [L, N, D]
  float *gh, *gz2, *gz1, *gaggr;         // backward temporaries
  float* wimg;                           // per layer: the weight images of the 2D-row and the D-row B operand (GinImages)
};

// The weight images of the MLP GEMMs (dense_tc.cu: each weight split into tf32 hi / lo once, in the layout of the GEMM's
// shared-memory stage).  The forward packs mlp.0.weight and mlp.2.weight as they are, the backward their transposes (the dgrad B
// operands), into the same workspace region: each pass packs its own, in one launch before its first GEMM.  Per layer the image
// with 2D rows comes first (mlp.0.weight forward, mlp.2.weight^T backward; reduction D), then the one with D rows (reduction 2D).
inline int64_t gin_image_floats(int64_t D) { return pgnn_tc_image_floats(2 * D, D) + pgnn_tc_image_floats(D, 2 * D); }

GinWs carve_gin(void* base, int64_t N, int64_t E, int64_t L, int64_t D) {
  Carve c(base);
  GinWs w;
  carve_front(c, w, false, kGin, N, E, D);
  w.bn_acc = c.take<double>(L * 2 * D);
  w.scale = c.take<float>(L * D);
  w.shift = c.take<float>(L * D);
  w.mean = c.take<float>(L * D);
  w.invstd = c.take<float>(L * D);
  w.aggr = c.take<float>(L * N * D);
  w.z1 = c.take<float>(L * N * 2 * D);
  w.z2 = c.take<float>(L * N * D);
  w.gh = c.take<float>(N * D);
  w.gz2 = c.take<float>(2 * N * D);       // two copies each: layer l's weight-gradient GEMMs (side stream) may still read
  w.gz1 = c.take<float>(2 * N * 2 * D);   // them while layer l-1's backward writes the other copy
  w.gaggr = c.take<float>(N * D);
  w.wimg = c.take<float>(L * gin_image_floats(D));
  carve_tail(c, w, kGin, N, E, D, split_k_floats(N, 2 * D, D), D);  // both MLP weight gradients have 2D*D elements
  return w;
}

// GCN / GraphSAGE / GAT of both domains; C = the Linear's width (H*D for GAT), Q = the summary's columns
struct ConvWs : Front, Tail {
  float *T, *xl, *z, *hout;    // [L][Q][C] tables (bio; chem GAT); per layer: Linear output [N, C], conv output [N, D], layer output [N, D]
  float *nrm, *alpha, *pq;     // per layer: SAGE row norms [N]; GAT attention [(E+N), H] and logit halves [N, H, 2]
  float *mean, *invstd;        // chem: BatchNorm batch statistics [L, D]
  float *gz, *ga, *gxl, *gh;   // backward temporaries [N, D], [N, D], two copies of [N, C] by layer parity, [N, D]
  float* gT;                   // bio: table gradients [L][Q][C]
};

ConvWs carve_conv(void* base, bool bio, int type, int64_t N, int64_t E, int64_t L, int64_t D) {
  Carve c(base);
  ConvWs w;
  const bool gat = type == PGNN_CONV_GAT;
  const int64_t C = gat ? kHeads * D : D, Q = bio ? kBioQ : kChemQ;
  carve_front(c, w, bio, type, N, E, D);
  w.T = c.take<float>(bio || gat ? L * Q * C : 0);
  w.xl = c.take<float>(L * N * C);
  w.z = c.take<float>(L * N * D);
  w.hout = c.take<float>(L * N * D);
  w.nrm = c.take<float>(type == PGNN_CONV_SAGE ? L * N : 0);
  w.alpha = c.take<float>(gat ? L * (E + N) * kHeads : 0);
  w.pq = c.take<float>(gat ? L * N * kHeads * 2 : 0);
  w.mean = c.take<float>(bio ? 0 : L * D);
  w.invstd = c.take<float>(bio ? 0 : L * D);
  w.gz = c.take<float>(N * D);
  w.ga = c.take<float>(N * D);
  w.gxl = c.take<float>(2 * N * C);   // two copies by layer parity: the side-stream wgrad of layer l reads one while layer l-1 writes the other
  w.gh = c.take<float>(N * D);
  w.gT = c.take<float>(bio ? L * Q * C : 0);
  carve_tail(c, w, type, N, E, D, bio ? pgnn_tc_wgrad_workspace_floats(N, C, D) : split_k_floats(N, C, D), bio ? 0 : D);
  return w;
}

// A tensor-path GEMM's weight operand as an image: its base, padded row count and row stride.  w == nullptr: no image.
struct Img {
  const float* w = nullptr;
  int64_t rows = 0, k = 0;
};

struct GinImages {
  const float* base = nullptr;  // nullptr: the GEMMs read the raw weights (more than 16 layers, precision 0)
  int64_t D = 0;
  Img wide(int64_t l) const { return base ? Img{base + l * gin_image_floats(D), align_up(2 * D, 128), align_up(D, 32)} : Img{}; }
  Img narrow(int64_t l) const {
    return base ? Img{base + l * gin_image_floats(D) + pgnn_tc_image_floats(2 * D, D), align_up(D, 128), align_up(2 * D, 32)} : Img{};
  }
};

int pack_gin_images(const GinWs& w, const void* const* params, int64_t L, int64_t D, bool transposed, cudaStream_t st, GinImages& im) {
  im = GinImages{};
  const char* e = getenv("PGNN_WEIGHT_IMAGES");  // =0: the raw-weight GEMMs, for comparing the two paths
  if (2 * L > 32 || (e && e[0] == '0')) return PGNN_OK;
  const float* src[32];
  float* dst[32];
  int64_t ld[32];
  int rows[32], cols[32], tr[32];
  for (int64_t l = 0; l < L; ++l) {
    const void* const* p = params + P_LAYER0 + l * L_COUNT;
    const float* w1 = (const float*)p[L_W1];  // [2D, D]
    const float* w2 = (const float*)p[L_W2];  // [D, 2D]
    const int i = (int)(2 * l);
    src[i] = transposed ? w2 : w1;      // 2D rows
    src[i + 1] = transposed ? w1 : w2;  // D rows
    dst[i] = w.wimg + l * gin_image_floats(D);
    dst[i + 1] = dst[i] + pgnn_tc_image_floats(2 * D, D);
    rows[i] = (int)(transposed ? D : 2 * D);
    cols[i] = (int)(transposed ? 2 * D : D);
    rows[i + 1] = (int)(transposed ? 2 * D : D);
    cols[i + 1] = (int)(transposed ? D : 2 * D);
    ld[i] = cols[i];
    ld[i + 1] = cols[i + 1];
    tr[i] = tr[i + 1] = transposed ? 1 : 0;
  }
  const int rc = pgnn_internal_pack_images((int)(2 * L), src, ld, rows, cols, tr, dst, st);
  if (rc == PGNN_OK) im = GinImages{w.wimg, D};
  else if (rc != PGNN_EUNSUPPORTED) return rc;
  return PGNN_OK;
}

// The forward GEMM y = act(x W^T + b) and the dgrad GEMM gx = (gy W) masked by relu_src > 0, each through the first path that
// covers it: the weight image when there is one, the raw-weight tensor path (precision 1), the generic pgnn_linear_*.  Only the
// tensor paths run the epilogue hooks `hk`; *hooked (when given) says whether one did.
int linear_fwd(const Img& im, const float* x, int64_t ldx, const float* W, const float* b, int64_t M, int64_t N, int64_t K, int relu,
               float* y, int64_t ldy, int precision, cudaStream_t st, const PgnnGemmHooks* hk = nullptr, bool* hooked = nullptr) {
  int rc = PGNN_EUNSUPPORTED;
  if (im.w) rc = pgnn_tc_linear_fwd_img(x, ldx, im.w, im.rows, im.k, b, M, N, K, relu, y, ldy, st, hk);
  if (rc == PGNN_EUNSUPPORTED && precision == 1) rc = pgnn_tc_linear_fwd(x, ldx, W, b, M, N, K, relu, y, ldy, st, hk);
  if (hooked) *hooked = rc == PGNN_OK;
  if (rc == PGNN_EUNSUPPORTED) rc = pgnn_linear_fwd(x, ldx, W, b, M, N, K, relu, y, ldy, precision, st);
  return rc;
}

int linear_bwd_x(const Img& im, const float* gy, int64_t ldgy, const float* W, int64_t M, int64_t N, int64_t K, const float* relu_src,
                 int64_t ldr, float* gx, int64_t ldgx, int precision, cudaStream_t st, const PgnnGemmHooks* hk, bool* hooked) {
  int rc = PGNN_EUNSUPPORTED;
  if (im.w) rc = pgnn_tc_linear_bwd_x_img(gy, ldgy, im.w, im.rows, im.k, M, N, K, relu_src, ldr, gx, ldgx, st, hk);
  if (rc == PGNN_EUNSUPPORTED && precision == 1) rc = pgnn_tc_linear_bwd_x(gy, ldgy, W, M, N, K, relu_src, ldr, gx, ldgx, st, hk);
  *hooked = rc == PGNN_OK;
  if (rc == PGNN_EUNSUPPORTED) rc = pgnn_linear_bwd_x(gy, ldgy, W, M, N, K, relu_src, ldr, gx, ldgx, precision, st);
  return rc;
}

// A Linear (no ReLU) whose tensor-path epilogue also accumulates the BatchNorm batch sums of y into acc [2][N] (fp64 atomics on
// a zeroed acc).  acc == nullptr, precision 0 or a shape no tensor path covers: a plain Linear with fused = false, and the
// caller computes the statistics itself.
int linear_bn_stats(double* acc, const Img& im, const float* x, int64_t ldx, const float* W, const float* b, int64_t M, int64_t N,
                    int64_t K, float* y, int64_t ldy, int precision, cudaStream_t st, bool& fused) {
  fused = false;
  if (!acc || precision != 1) return linear_fwd(im, x, ldx, W, b, M, N, K, 0, y, ldy, precision, st);
  PGNN_CUDA(cudaMemsetAsync(acc, 0, sizeof(double) * 2 * N, st));
  PgnnGemmHooks hk;
  hk.stats = acc;
  return linear_fwd(im, x, ldx, W, b, M, N, K, 0, y, ldy, precision, st, &hk, &fused);
}

// The finalisation of layer l's BatchNorm from the sums a fused Linear left in acc, for the consumer kernel that applies it: it
// also updates the running state and saves the batch mean / invstd for the backward.
PgnnBnFold bn_fold(const BnRun& bn, int64_t l, double* acc, const float* gamma, const float* beta, float* save_mean, float* save_invstd,
                   int64_t rows) {
  PgnnBnFold f{};
  f.acc = acc; f.gamma = gamma; f.beta = beta;
  f.running_mean = bn.rm(l); f.running_var = bn.rv(l); f.nbt = bn.nb(l);
  f.save_mean = save_mean; f.save_invstd = save_invstd;
  f.momentum = bn.momentum; f.eps = bn.eps; f.set_rows((int)rows);
  return f;
}

// Weight-gradient GEMMs on a side stream.  They only feed the gradient buffer, so on their own stream they run under the next
// layer's BatchNorm sweeps, attention and gathers (LSU / L2-bound kernels that leave the tensor pipe and most of shared memory
// idle) instead of in front of them.  One context per (device, main stream) serves every type; PGNN_WGRAD_STREAM=0 disables.
// The operands are double-buffered by layer parity so the main stream never overwrites one a pending wgrad still reads.  Event
// pair k (GIN: 0 = the wgrad of the layer's last Linear, 1 = of its first; the conv types: 0) of parity par orders them:
//   - before it writes layer l's operand of wgrad k, the main stream waits for done[k][l & 1] (layer l+2's wgrad k is through);
//   - side_wgrad records ready[k][l & 1] on the main stream, and the side stream waits for it before the wgrad;
//   - the side stream records done[k][l & 1] after it;
//   - a wgrad the tensor path does not cover joins the side stream into the main stream and runs there;
//   - every backward joins the side stream into the main stream before the embedding gradients (join_side).
struct SideCtx {
  cudaStream_t side = nullptr;
  cudaEvent_t ready[2][2] = {}, done[2][2] = {}, join = nullptr;
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
  for (int k = 0; k < 2 && ok; ++k)
    for (int i = 0; i < 2 && ok; ++i)
      ok = cudaEventCreateWithFlags(&c->ready[k][i], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&c->done[k][i], cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&c->join, cudaEventDisableTiming) == cudaSuccess;
  if (!ok) cudaGetLastError();
  c->ok = ok;
  return ok ? c : nullptr;
}

// the main stream waits for everything enqueued on the side stream so far
int join_side(const SideCtx* sc, cudaStream_t st) {
  PGNN_CUDA(cudaEventRecord(sc->join, sc->side));
  PGNN_CUDA(cudaStreamWaitEvent(st, sc->join, 0));
  return PGNN_OK;
}

// the main stream waits until layer l+2's wgrad k has finished reading the operand copy of parity par
int side_wait(const SideCtx* sc, cudaStream_t st, int k, int par) {
  if (sc) PGNN_CUDA(cudaStreamWaitEvent(st, sc->done[k][par], 0));
  return PGNN_OK;
}

// One weight-gradient GEMM: gw [Nout, K] = gy^T x and gb = the column sums of gy (gb may be null), ordered as SideCtx describes
int side_wgrad(const SideCtx* sc, cudaStream_t st, int k, int par, int precision, const float* gy, int64_t ldgy, const float* x,
               int64_t ldx, int64_t M, int64_t Nout, int64_t K, float* gw, float* gb, float* wpart, int64_t wpart_floats) {
  cudaStream_t wst = sc ? sc->side : st;
  if (sc) {
    PGNN_CUDA(cudaEventRecord(sc->ready[k][par], st));
    PGNN_CUDA(cudaStreamWaitEvent(wst, sc->ready[k][par], 0));
  }
  int rc = PGNN_EUNSUPPORTED;
  if (precision == 1) rc = pgnn_tc_linear_bwd_w_ws(gy, ldgy, x, ldx, M, Nout, K, gw, gb, wpart, wpart_floats, wst);
  if (rc == PGNN_EUNSUPPORTED) {
    if (sc) TRY(join_side(sc, st));
    return pgnn_linear_bwd_w(gy, ldgy, x, ldx, M, Nout, K, gw, gb, precision, st);
  }
  if (rc == PGNN_OK && sc) PGNN_CUDA(cudaEventRecord(sc->done[k][par], wst));
  return rc;
}

// Graph preparation, the per-node bond summary S (not for GAT, whose kernels read the bond codes per edge), the atom embedding
// and, for the tensor-path backward, the one-hot atom-code rows.
int forward_prologue(int type, const Front& f, const void* const* params, const int64_t* x, const int64_t* edge_index,
                     const int64_t* edge_attr, int64_t N, int64_t E, int64_t D, int training, int precision, void* scratch,
                     int64_t scratch_bytes, cudaStream_t st) {
  TRY(pgnn_graph_prep(edge_index, E, N, f.rowptr_t, f.nbr_t, f.eid_t, f.rowptr_s, f.nbr_s, f.eid_s, scratch, scratch_bytes, st));
  if (type == PGNN_CONV_GCN) TRY(pgnn_gcn_dinv(f.rowptr_t, N, f.dinv, st));
  if (type != PGNN_CONV_GAT) TRY(pgnn_chem_edge_summary(edge_attr, f.rowptr_t, f.nbr_t, f.eid_t, N, agg_mode(type), f.dinv, f.S, st));
  TRY(pgnn_chem_embed_fwd(x, (const float*)params[P_XEMB1], kAtomRows, (const float*)params[P_XEMB2], kChiralRows, N, D, f.h0, D, st));
  if (training && precision == 1) TRY(pgnn_internal_chem_onehot(x, N, kAtomRows, kChiralRows, f.onehot, kOneHotLd, st));
  return PGNN_OK;
}

// Backward tail of every chem type: the side stream's last wgrad (and its use of the split-K workspace) joins the main stream,
// then the embedding tables: [120 + 3, D] = onehot^T . gh as a split-K weight-gradient GEMM (the two tables are adjacent in the
// flat layout); the vector-atomics kernel is the FFMA-precision path and the fallback.
int embed_backward(const SideCtx* sc, const Front& f, const float* gh, const int64_t* x, int64_t N, int64_t D, int precision,
                   float* grads, const int64_t* off, float* wpart, int64_t wpart_floats, cudaStream_t st) {
  if (sc) TRY(join_side(sc, st));
  int rc = PGNN_EUNSUPPORTED;
  if (precision == 1)
    rc = pgnn_tc_linear_bwd_w_ws(f.onehot, kOneHotLd, gh, D, N, kAtomRows + kChiralRows, D, grads + off[P_XEMB1], nullptr, wpart,
                                 wpart_floats, st);
  if (rc == PGNN_EUNSUPPORTED)
    rc = pgnn_chem_embed_bwd(x, gh, D, N, D, grads + off[P_XEMB1], kAtomRows, grads + off[P_XEMB2], kChiralRows, st);
  return rc;
}

int gin_forward(const void* const* params, const BnRun& bn, int training, const Drops& drops, int precision, float* node_rep,
                int64_t ld_out, int64_t N, int64_t L, int64_t D, const GinWs& w, cudaStream_t st) {
  GinImages im;
  if (precision == 1) TRY(pack_gin_images(w, params, L, D, false, st, im));
  const float* h = w.h0;            // input rows of the current layer (pre-affine)
  const float *in_scale = nullptr, *in_shift = nullptr;
  PgnnBnFold fold;                  // pending BatchNorm finalisation of the previous layer (folded into this layer's gather)
  bool have_fold = false;
  for (int64_t l = 0; l < L; ++l) {
    const void* const* p = params + P_LAYER0 + l * L_COUNT;
    float* aggr = w.aggr + l * N * D;
    float* z1 = w.z1 + l * N * 2 * D;
    float* z2 = w.z2 + l * N * D;
    const bool last = (l == L - 1);
    const PgnnDropout drop_in = drops.at(l > 0 ? l - 1 : 0), drop_out = drops.at(l);  // the previous layer's mask, this layer's
    // gather (the previous layer's BatchNorm + ReLU + dropout applied on load) + GEMM1
    TRY(pgnn_internal_aggregate_fwd(h, D, in_scale, in_shift, in_scale != nullptr || have_fold, N, D, w.rowptr_t, w.nbr_t, PGNN_AGG_SUM,
                                    nullptr, w.S, kChemQ, (const float*)p[L_ET1], (const float*)p[L_ET2], kChemQSplit, 0, aggr, D, st,
                                    have_fold ? &fold : nullptr, l > 0 ? &drop_in : nullptr));
    TRY(linear_fwd(im.wide(l), aggr, D, (const float*)p[L_W1], (const float*)p[L_B1], N, 2 * D, D, 1, z1, 2 * D, precision, st));
    have_fold = false;
    // GEMM2; in training on the tensor path its epilogue also accumulates the BatchNorm batch statistics of z2
    double* acc = w.bn_acc + l * 2 * D;
    bool stats_fused;
    TRY(linear_bn_stats(training ? acc : nullptr, im.narrow(l), z1, 2 * D, (const float*)p[L_W2], (const float*)p[L_B2], N, D, 2 * D, z2, D,
                        precision, st, stats_fused));
    if (stats_fused) {
      // no finalize launch: the consumer (next layer's gather, or the final apply) derives scale/shift from the sums
      fold = bn_fold(bn, l, acc, (const float*)p[L_GAMMA], (const float*)p[L_BETA], w.mean + l * D, w.invstd + l * D, N);
      if (last) {
        TRY(pgnn_internal_bn_apply_fold(z2, D, N, D, fold, 0, node_rep, ld_out, st, &drop_out));
      } else {
        have_fold = true;
      }
      h = z2;
      in_scale = in_shift = nullptr;
    } else if (training) {
      // statistics only for inner layers (applied on load by the next gather); the last layer materialises node_rep
      TRY(pgnn_internal_bn_fwd_train(z2, D, N, D, (const float*)p[L_GAMMA], (const float*)p[L_BETA], bn.rm(l), bn.rv(l), bn.nb(l),
                                     bn.momentum, bn.eps, 0, last ? node_rep : nullptr, ld_out, w.mean + l * D, w.invstd + l * D,
                                     w.scale + l * D, w.shift + l * D, w.scratch, w.scratch_bytes, st, &drop_out));
      h = z2;
      in_scale = w.scale + l * D;
      in_shift = w.shift + l * D;
    } else {
      // eval: plain BN(+ReLU) pass with the running statistics, ping-ponging between two spare buffers
      float* y = last ? node_rep : ((l & 1) ? w.gz2 : w.gaggr);
      TRY(pgnn_bn_fwd_eval(z2, D, N, D, (const float*)p[L_GAMMA], (const float*)p[L_BETA], bn.rm(l), bn.rv(l), bn.eps, !last, y,
                           last ? ld_out : D, st));
      h = y;
      in_scale = in_shift = nullptr;
    }
  }
  return PGNN_OK;
}

int gin_backward(const void* const* params, const float* g_node_rep, int64_t ldg, const int64_t* x, int64_t N, int64_t L, int64_t D,
                 const Drops& drops, int precision, float* grads, const int64_t* off, const GinWs& w, cudaStream_t st) {
  // images of the transposed MLP weights: the dgrad B operands, reduction-contiguous and already split
  GinImages im;
  if (precision == 1) TRY(pack_gin_images(w, params, L, D, true, st, im));
  const float* gy = g_node_rep;
  int64_t ldgy = ldg;
  SideCtx* sc = precision == 1 ? side_ctx(st) : nullptr;
  for (int64_t l = L - 1; l >= 0; --l) {
    const void* const* p = params + P_LAYER0 + l * L_COUNT;
    const int64_t* o = off + P_LAYER0 + l * L_COUNT;
    const float* aggr = w.aggr + l * N * D;
    const float* z1 = w.z1 + l * N * 2 * D;
    const float* z2 = w.z2 + l * N * D;
    const bool last = (l == L - 1);
    const int par = (int)(l & 1);
    float* gz2 = w.gz2 + (sc ? par * N * D : 0);
    float* gz1 = w.gz1 + (sc ? par * N * 2 * D : 0);
    // BatchNorm (dropout mask regenerated, ReLU mask recomputed from z2) backward; the same pass leaves colsum(gz2) = gradient
    // of mlp.2.bias
    TRY(side_wait(sc, st, 0, par));
    const PgnnDropout drop = drops.at(l);
    TRY(pgnn_internal_bn_bwd(gy, ldgy, z2, D, N, D, (const float*)p[L_GAMMA], (const float*)p[L_BETA], w.mean + l * D,
                             w.invstd + l * D, !last, gz2, D, grads + o[L_GAMMA], grads + o[L_BETA], grads + o[L_B2],
                             w.scratch, w.scratch_bytes, st, &drop));
    // MLP backward.  On the tensor path the dgrad epilogues carry the column reductions that would otherwise be passes of
    // their own: colsum(gz1) = gradient of mlp.0.bias, and S^T gaggr = gradient of the two bond tables.  Where a dgrad falls
    // back, wgrad1 computes the bias gradient and a separate pass the tables'.
    TRY(side_wgrad(sc, st, 0, par, precision, gz2, D, z1, 2 * D, N, D, 2 * D, grads + o[L_W2], nullptr, w.wpart, w.wpart_floats));
    TRY(side_wait(sc, st, 1, par));
    PGNN_CUDA(cudaMemsetAsync(grads + o[L_B1], 0, sizeof(float) * 2 * D, st));
    PgnnGemmHooks h1;
    h1.colsum = grads + o[L_B1];
    bool b1_done;
    TRY(linear_bwd_x(im.wide(l), gz2, D, (const float*)p[L_W2], N, D, 2 * D, z1, 2 * D, gz1, 2 * D, precision, st, &h1, &b1_done));
    TRY(side_wgrad(sc, st, 1, par, precision, gz1, 2 * D, aggr, D, N, 2 * D, D, grads + o[L_W1], b1_done ? nullptr : grads + o[L_B1],
                   w.wpart, w.wpart_floats));
    PGNN_CUDA(cudaMemsetAsync(grads + o[L_ET1], 0, sizeof(float) * kChemQ * D, st));  // the two tables are adjacent in the layout
    PgnnGemmHooks h2;
    h2.S = w.S; h2.Q = kChemQ; h2.gT = grads + o[L_ET1]; h2.gT2 = grads + o[L_ET2]; h2.q_split = kChemQSplit; h2.ldt = D;
    bool et_done;
    TRY(linear_bwd_x(im.narrow(l), gz1, 2 * D, (const float*)p[L_W1], N, 2 * D, D, nullptr, 0, w.gaggr, D, precision, st, &h2, &et_done));
    if (!et_done)
      TRY(pgnn_internal_edge_table_bwd2(w.S, kChemQ, w.gaggr, D, 0, N, (int)D, grads + o[L_ET1], D, grads + o[L_ET2], kChemQSplit, st));
    // transpose-graph gather: gradient w.r.t. this layer's input rows
    TRY(pgnn_aggregate_bwd(w.gaggr, D, N, D, w.rowptr_s, w.nbr_s, PGNN_AGG_SUM, nullptr, w.rowptr_t, w.gh, D, st));
    gy = w.gh;
    ldgy = D;
  }
  return embed_backward(sc, w, w.gh, x, N, D, precision, grads, off, w.wpart, w.wpart_floats, st);
}

// ==============================================================================================================================
// bio (bio/model.py:11-290 with JK="last", any drop_ratio)
// ==============================================================================================================================
// Layer 0 embeds the dummy node label (input_node_embeddings [2, D]).  Each conv's edge encoder Linear(9, C) acts through the
// per-node summary S [N, 10] (pgnn_bio_edge_summary) and the table T [10, C] = [W^T ; b]: the forward packs every layer's table in
// one launch, and the backward scatters every layer's table gradient back as the encoder's weight [C, 9] and bias [C] in one.
//   GIN        aggr = [sum_j x_j || S.T] (2D wide), then Linear(2D,2D) -> BatchNorm1d(2D) -> ReLU -> Linear(2D,D)
//   GCN / GraphSAGE / GAT: the chem layer body (conv_forward / conv_backward) with the bio table (GAT reads the 9 float
//              attributes per edge).
// There is no outer BatchNorm: every layer but the last is followed by ReLU, then by layer l's dropout mask.  GIN applies both on
// load in the next layer's gather (and, under dropout, its last layer takes one dropout sweep that writes node_rep); the conv
// types take one ReLU + dropout sweep per layer that writes the layer's output (bio_act).  The backward runs the matching sweep
// on the incoming gradient of every layer.

constexpr int kBioEmbRows = 2;  // input_node_embeddings
constexpr int kMaxPack = 64;    // layers per table-pack launch (their pointers travel as kernel arguments)

// order of the bio parameter pointer table and of its flat gradient layout (one enum, so the types' indices mix in expressions)
enum BioParam {
  PB_EMB = 0, PB_LAYER0 = 1,
  BG_W1 = 0, BG_B1, BG_GAMMA, BG_BETA, BG_W2, BG_B2, BG_ENC_W, BG_ENC_B, BG_COUNT,  // gin: mlp.0, mlp.1, mlp.3, edge_encoder
  BC_W = 0, BC_B, BC_ENC_W, BC_ENC_B, BC_COUNT,                                     // gcn / graphsage
  BA_W = 0, BA_B, BA_ATT, BA_BIAS, BA_ENC_W, BA_ENC_B, BA_COUNT                     // gat
};
static_assert(BC_W == CV_W && BC_B == CV_B && BA_W == CV_W && BA_B == CV_B && BA_ATT == CV_ATT && BA_BIAS == CV_BIAS, "bio conv order");

inline int bio_layer_params(int type) { return type == kGin ? BG_COUNT : type == PGNN_CONV_GAT ? BA_COUNT : BC_COUNT; }
inline int bio_enc_w(int type) { return type == kGin ? BG_ENC_W : type == PGNN_CONV_GAT ? BA_ENC_W : BC_ENC_W; }
inline int64_t bio_width(int type, int64_t D) { return type == PGNN_CONV_GAT ? kHeads * D : D; }  // C: the edge encoder's width

int64_t bio_grad_layout(int type, int64_t L, int64_t D, int64_t* offsets) {
  if (!offsets) return 1 + (int64_t)bio_layer_params(type) * L;
  const int64_t C = bio_width(type, D);
  int64_t o = 0, i = 0;
  auto next = [&](int64_t size) { offsets[i++] = o; o += size; };
  next(kBioEmbRows * D);  // gnns.0.input_node_embeddings.weight
  for (int64_t l = 0; l < L; ++l) {
    if (type == kGin) {
      next(4 * D * D);  // mlp.0.weight [2D, 2D]
      next(2 * D);      // mlp.0.bias
      next(2 * D);      // mlp.1.weight (BatchNorm1d(2D))
      next(2 * D);      // mlp.1.bias
      next(2 * D * D);  // mlp.3.weight [D, 2D]
      next(D);          // mlp.3.bias
    } else {
      next(C * D);  // linear.weight / weight_linear.weight [C, D]
      next(C);      // its bias
      if (type == PGNN_CONV_GAT) {
        next(kHeads * 2 * D);  // att [1, H, 2D]
        next(D);               // bias [D]
      }
    }
    next(9 * C);  // edge_encoder.weight [C, 9]
    next(C);      // edge_encoder.bias (adjacent: the table gradient scatter writes both)
  }
  offsets[i] = o;
  return i;
}

struct PackArgs {
  const float* w[kMaxPack];
  const float* b[kMaxPack];
};

// T[l][q][c] = W_l[c][q] for q < 9, T[l][9][c] = b_l[c]: `count` layers' edge encoders as the [10, C] tables the kernels index
__global__ void __launch_bounds__(256) k_bio_pack_tables(PackArgs a, int count, int C, float* __restrict__ T) {
  pdl_prologue();
  const int64_t per = (int64_t)kBioQ * C, total = per * count;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int l = (int)(idx / per);
    const int r = (int)(idx - l * per);
    const int q = r / C, c = r - q * C;
    T[idx] = q < 9 ? a.w[l][c * 9 + q] : a.b[l][c];
  }
}

// the transpose: gT [L][10][C] -> every layer's edge_encoder.weight [C, 9] and .bias [C] gradients, layer l's at out + l * stride
__global__ void __launch_bounds__(256) k_bio_unpack_table_grads(const float* __restrict__ gT, int64_t L, int C, float* __restrict__ out,
                                                                int64_t stride) {
  pdl_prologue();
  const int64_t per = (int64_t)kBioQ * C, total = per * L;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = idx / per;
    const int r = (int)(idx - l * per);
    const int q = r / C, c = r - q * C;
    out[l * stride + (q < 9 ? (int64_t)c * 9 + q : (int64_t)9 * C + c)] = gT[idx];
  }
}

// The inter-layer activation of bio/model.py:278-286 as one sweep.  Forward (BWD = false): y = relu(x) (relu != 0; NaN kept)
// times layer d.layer's dropout factor.  Backward (BWD = true): gx = (relu ? (z > 0 ? gy : 0) : gy) times the same factor, z the
// forward's pre-activation.  DROP = false has no hash.  One warp per row, VEC (4: float4, 1: scalar, for strides that are not a
// multiple of 4) columns per lane.
__device__ __forceinline__ float bio_act1(float v, float z, bool bwd, int relu) {
  return relu ? (bwd ? (z > 0.f ? v : 0.f) : relu_keep_nan(v)) : v;
}

template <bool BWD, bool DROP, int VEC>
__global__ void __launch_bounds__(256) k_bio_act(const float* __restrict__ x, int64_t ldx, const float* __restrict__ z, int64_t ldz,
                                                 int64_t M, int64_t C, int relu, PgnnDropout d, float* __restrict__ y, int64_t ldy) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); r < M; r += warps) {
    for (int64_t c = (int64_t)lane * VEC; c < C; c += 32 * VEC) {
      if (VEC == 4) {
        float4 v = ld4(x + r * ldx + c);
        const float4 zz = BWD && relu ? ld4(z + r * ldz + c) : v;
        v.x = bio_act1(v.x, zz.x, BWD, relu);
        v.y = bio_act1(v.y, zz.y, BWD, relu);
        v.z = bio_act1(v.z, zz.z, BWD, relu);
        v.w = bio_act1(v.w, zz.w, BWD, relu);
        if (DROP) v = dropout4(v, d, r, C, c);
        st4(y + r * ldy + c, v);
      } else {
        float v = bio_act1(x[r * ldx + c], BWD && relu ? z[r * ldz + c] : 0.f, BWD, relu);
        if (DROP) v *= dropout_factor(d, r, C, c);
        y[r * ldy + c] = v;
      }
    }
  }
}

int bio_act(bool bwd, const float* x, int64_t ldx, const float* z, int64_t ldz, int64_t M, int64_t C, int relu, const PgnnDropout& d,
            float* y, int64_t ldy, cudaStream_t st) {
  const bool drop = d.p > 0.f;
  const bool v4 = C % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0 && aligned16(x) && aligned16(y) &&
                  (!(bwd && relu) || (ldz % 4 == 0 && aligned16(z)));
  auto k = v4 ? (bwd ? (drop ? k_bio_act<true, true, 4> : k_bio_act<true, false, 4>) : (drop ? k_bio_act<false, true, 4> : k_bio_act<false, false, 4>))
              : (bwd ? (drop ? k_bio_act<true, true, 1> : k_bio_act<true, false, 1>) : (drop ? k_bio_act<false, true, 1> : k_bio_act<false, false, 1>));
  PGNN_CUDA(pgnn_launch(k, dim3(grid_items(M * 32, 256)), dim3(256), 0, st, x, ldx, z, ldz, M, C, relu, d, y, ldy));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

// the backward's gradient at layer l's pre-activation: the incoming rows themselves when the layer has neither ReLU nor dropout
// and the consumers can read them in place (16-byte rows), else the bio_act sweep into `buf`
int bio_act_bwd(const float*& gz, int64_t& ldgz, const float* gy, int64_t ldgy, const float* z, int64_t M, int64_t D, bool last,
                const PgnnDropout& d, float* buf, cudaStream_t st) {
  if (last && d.p == 0.f && ldgy % 4 == 0 && aligned16(gy)) {
    gz = gy;
    ldgz = ldgy;
    return PGNN_OK;
  }
  gz = buf;
  ldgz = D;
  return bio_act(true, gy, ldgy, z, D, M, D, !last, d, buf, D, st);
}

int bio_pack_tables(int type, const void* const* params, int64_t L, int64_t C, float* T, cudaStream_t st) {
  const int PL = bio_layer_params(type), ew = bio_enc_w(type);
  for (int64_t l0 = 0; l0 < L; l0 += kMaxPack) {
    const int count = (int)(L - l0 < kMaxPack ? L - l0 : kMaxPack);
    PackArgs a{};
    for (int i = 0; i < count; ++i) {
      const void* const* p = params + PB_LAYER0 + (l0 + i) * PL;
      a.w[i] = (const float*)p[ew];
      a.b[i] = (const float*)p[ew + 1];
      PGNN_CHECK_ARG(a.w[i] && a.b[i]);
    }
    PGNN_CUDA(pgnn_launch(k_bio_pack_tables, dim3(grid_items(kBioQ * C * count, 256)), dim3(256), 0, st, a, count, (int)C,
                          T + l0 * kBioQ * C));
    PGNN_LAUNCH_CHECK();
  }
  return PGNN_OK;
}

struct BioGinWs : Front, Tail {
  float* T;                      // [L][10][D] packed edge-encoder tables
  double* bn_acc;                // [L][2][2D] fp64 sums of the inner BatchNorm (tensor path)
  float *mean, *invstd;          // [L, 2D]
  float *aggr, *z1, *y1, *z2;    // per layer: gather [N, 2D], Linear 1 [N, 2D], BatchNorm + ReLU [N, 2D], Linear 2 [N, D]
  float *gz2, *gy1, *gz1, *ga;   // backward temporaries; gz2 and gz1 two copies by layer parity (side-stream wgrad operands)
  float *gh, *gT;                // [N, D], [L][10][D]
};

BioGinWs carve_bio_gin(void* base, int64_t N, int64_t E, int64_t L, int64_t D) {
  Carve c(base);
  BioGinWs w;
  const int64_t D2 = 2 * D;
  carve_front(c, w, true, kGin, N, E, D);
  w.T = c.take<float>(L * kBioQ * D);
  w.bn_acc = c.take<double>(L * 2 * D2);
  w.mean = c.take<float>(L * D2);
  w.invstd = c.take<float>(L * D2);
  w.aggr = c.take<float>(L * N * D2);
  w.z1 = c.take<float>(L * N * D2);
  w.y1 = c.take<float>(L * N * D2);
  w.z2 = c.take<float>(L * N * D);
  w.gz2 = c.take<float>(2 * N * D);
  w.gy1 = c.take<float>(N * D2);
  w.gz1 = c.take<float>(2 * N * D2);
  w.ga = c.take<float>(N * D2);
  w.gh = c.take<float>(N * D);
  w.gT = c.take<float>(L * kBioQ * D);
  const int64_t a = pgnn_tc_wgrad_workspace_floats(N, D2, D2), b = pgnn_tc_wgrad_workspace_floats(N, D, D2);
  carve_tail(c, w, kGin, N, E, D, a > b ? a : b, D2);
  return w;
}

// Graph preparation, the summary S (not for GAT, whose kernels read the attributes per edge), the label embedding and every
// layer's packed edge-encoder table.
int bio_prologue(int type, const Front& f, float* T, const void* const* params, const float* x, const int64_t* edge_index,
                 const float* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D, void* scratch, int64_t scratch_bytes, cudaStream_t st) {
  TRY(pgnn_graph_prep(edge_index, E, N, f.rowptr_t, f.nbr_t, f.eid_t, f.rowptr_s, f.nbr_s, f.eid_s, scratch, scratch_bytes, st));
  if (type == PGNN_CONV_GCN) TRY(pgnn_gcn_dinv(f.rowptr_t, N, f.dinv, st));
  if (type != PGNN_CONV_GAT) TRY(pgnn_bio_edge_summary(edge_attr, f.rowptr_t, f.nbr_t, f.eid_t, N, agg_mode(type), f.dinv, f.S, st));
  TRY(pgnn_bio_embed_fwd(x, (const float*)params[PB_EMB], N, D, f.h0, D, st));
  return bio_pack_tables(type, params, L, bio_width(type, D), T, st);
}

// Backward tail of every bio type: the side stream joins, then the label-embedding gradient and the edge-encoder gradients of
// every layer from the table gradients gT [L][10][C].
int bio_backward_tail(int type, const SideCtx* sc, const float* gT, const float* gh, const float* x, int64_t N, int64_t L, int64_t D,
                      float* grads, const int64_t* off, cudaStream_t st) {
  if (sc) TRY(join_side(sc, st));
  TRY(pgnn_bio_embed_bwd(x, gh, D, N, D, grads + off[PB_EMB], st));
  const int64_t C = bio_width(type, D);
  const int64_t stride = off[PB_LAYER0 + bio_layer_params(type)] - off[PB_LAYER0];
  PGNN_CUDA(pgnn_launch(k_bio_unpack_table_grads, dim3(grid_items(L * kBioQ * C, 256)), dim3(256), 0, st, gT, L, (int)C,
                        grads + off[PB_LAYER0 + bio_enc_w(type)], stride));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int bio_gin_forward(const void* const* params, const BnRun& bn, int64_t N, int64_t L, int64_t D, int training, const Drops& drops,
                    int precision, float* node_rep, int64_t ld_out, const BioGinWs& w, cudaStream_t st) {
  const int64_t D2 = 2 * D;
  for (int64_t l = 0; l < L; ++l) {
    const void* const* p = params + PB_LAYER0 + l * BG_COUNT;
    float* aggr = w.aggr + l * N * D2;
    float* z1 = w.z1 + l * N * D2;
    float* y1 = w.y1 + l * N * D2;
    float* z2 = w.z2 + l * N * D;
    const bool last = l == L - 1;
    const PgnnDropout drop_in = drops.at(l > 0 ? l - 1 : 0), drop_out = drops.at(l);
    // gather: columns 0..D the inputs (the previous layer's ReLU + dropout applied on load), D..2D the edge-encoder half S.T
    const float* h = l == 0 ? w.h0 : w.z2 + (l - 1) * N * D;
    TRY(pgnn_internal_aggregate_fwd(h, D, nullptr, nullptr, l > 0, N, D, w.rowptr_t, w.nbr_t, PGNN_AGG_SUM, nullptr, w.S, kBioQ,
                                    w.T + l * kBioQ * D, nullptr, kBioQ, D, aggr, D2, st, nullptr, l > 0 ? &drop_in : nullptr));
    // Linear 1; on the tensor path in training its epilogue also accumulates the inner BatchNorm's batch statistics
    const float* gamma = (const float*)p[BG_GAMMA];
    const float* beta = (const float*)p[BG_BETA];
    double* acc = w.bn_acc + l * 2 * D2;
    bool stats_fused;
    TRY(linear_bn_stats(training ? acc : nullptr, Img{}, aggr, D2, (const float*)p[BG_W1], (const float*)p[BG_B1], N, D2, D2, z1, D2,
                        precision, st, stats_fused));
    // inner BatchNorm1d(2D) + ReLU
    if (stats_fused) {
      const PgnnBnFold fold = bn_fold(bn, l, acc, gamma, beta, w.mean + l * D2, w.invstd + l * D2, N);
      TRY(pgnn_internal_bn_apply_fold(z1, D2, N, D2, fold, 1, y1, D2, st, nullptr));
    } else if (training) {
      TRY(pgnn_internal_bn_fwd_train(z1, D2, N, D2, gamma, beta, bn.rm(l), bn.rv(l), bn.nb(l), bn.momentum, bn.eps, 1, y1, D2,
                                     w.mean + l * D2, w.invstd + l * D2, nullptr, nullptr, w.scratch, w.scratch_bytes, st, nullptr));
    } else {
      TRY(pgnn_bn_fwd_eval(z1, D2, N, D2, gamma, beta, bn.rm(l), bn.rv(l), bn.eps, 1, y1, D2, st));
    }
    // Linear 2: the layer's pre-activation; the last layer without dropout writes node_rep itself
    const bool direct = last && drop_out.p == 0.f;
    TRY(pgnn_linear_fwd(y1, D2, (const float*)p[BG_W2], (const float*)p[BG_B2], N, D, D2, 0, direct ? node_rep : z2, direct ? ld_out : D,
                        precision, st));
    if (last && !direct) TRY(bio_act(false, z2, D, nullptr, 0, N, D, 0, drop_out, node_rep, ld_out, st));
  }
  return PGNN_OK;
}

int bio_gin_backward(const void* const* params, const float* g_node_rep, int64_t ldg, const float* x, int64_t N, int64_t L, int64_t D,
                     const Drops& drops, int precision, float* grads, const int64_t* off, const BioGinWs& w, cudaStream_t st) {
  const int64_t D2 = 2 * D;
  SideCtx* sc = precision == 1 ? side_ctx(st) : nullptr;
  PGNN_CUDA(cudaMemsetAsync(w.gT, 0, sizeof(float) * L * kBioQ * D, st));
  const float* gy = g_node_rep;
  int64_t ldgy = ldg;
  for (int64_t l = L - 1; l >= 0; --l) {
    const void* const* p = params + PB_LAYER0 + l * BG_COUNT;
    const int64_t* o = off + PB_LAYER0 + l * BG_COUNT;
    const bool last = l == L - 1;
    const int par = (int)(l & 1);
    const float* aggr = w.aggr + l * N * D2;
    const float* z1 = w.z1 + l * N * D2;
    const float* y1 = w.y1 + l * N * D2;
    float* gz2 = w.gz2 + (sc ? par * N * D : 0);
    float* gz1 = w.gz1 + (sc ? par * N * D2 : 0);
    // the gradient at the layer's pre-activation: its ReLU (inner layers) and dropout masks in one sweep
    TRY(side_wait(sc, st, 0, par));
    const float* gz;
    int64_t ldgz;
    TRY(bio_act_bwd(gz, ldgz, gy, ldgy, w.z2 + l * N * D, N, D, last, drops.at(l), gz2, st));
    // Linear 2: weight and bias gradients (side stream), then the gradient of the BatchNorm's output
    TRY(side_wgrad(sc, st, 0, par, precision, gz, ldgz, y1, D2, N, D, D2, grads + o[BG_W2], grads + o[BG_B2], w.wpart, w.wpart_floats));
    TRY(pgnn_linear_bwd_x(gz, ldgz, (const float*)p[BG_W2], N, D, D2, nullptr, 0, w.gy1, D2, precision, st));
    // inner BatchNorm + ReLU (mask recomputed from z1); the same pass leaves colsum(gz1) = the gradient of mlp.0.bias
    TRY(side_wait(sc, st, 1, par));
    TRY(pgnn_internal_bn_bwd(w.gy1, D2, z1, D2, N, D2, (const float*)p[BG_GAMMA], (const float*)p[BG_BETA], w.mean + l * D2,
                             w.invstd + l * D2, 1, gz1, D2, grads + o[BG_GAMMA], grads + o[BG_BETA], grads + o[BG_B1], w.scratch,
                             w.scratch_bytes, st, nullptr));
    // Linear 1
    TRY(side_wgrad(sc, st, 1, par, precision, gz1, D2, aggr, D2, N, D2, D2, grads + o[BG_W1], nullptr, w.wpart, w.wpart_floats));
    TRY(pgnn_linear_bwd_x(gz1, D2, (const float*)p[BG_W1], N, D2, D2, nullptr, 0, w.ga, D2, precision, st));
    // the gather: gT_l = S^T ga[:, D:2D]; the node half goes back over the transpose graph
    TRY(pgnn_internal_edge_table_bwd2(w.S, kBioQ, w.ga, D2, D, N, (int)D, w.gT + l * kBioQ * D, D, nullptr, kBioQ, st));
    TRY(pgnn_aggregate_bwd(w.ga, D2, N, D, w.rowptr_s, w.nbr_s, PGNN_AGG_SUM, nullptr, w.rowptr_t, w.gh, D, st));
    gy = w.gh;
    ldgy = D;
  }
  return bio_backward_tail(kGin, sc, w.gT, w.gh, x, N, L, D, grads, off, st);
}

// ==============================================================================================================================
// GCN / GraphSAGE / GAT, both domains
// ==============================================================================================================================

// A conv layer's edge term.  The gathers read the summary S [N, Q] against the table T (rows < q_split) and T2 (the rest); GAT
// reads the one table T per edge, from the raw edge_attr as is_bio says.  The backward lands the table gradient on gT / gT2,
// zeroing them first when zero_gT (GAT's backward overwrites its own).
struct EdgeTerm {
  const float* S;
  int Q, q_split;
  const float *T, *T2;
  int is_bio;
  float *gT, *gT2;
  bool zero_gT;
};

// chem: the two bond tables (GAT: both in layer l's [9, C] workspace table, which the forward fills) and their gradients in the
// flat buffer; bio: layer l's packed [10, C] table and its gradient, zeroed once per pass and unpacked by bio_backward_tail
EdgeTerm edge_term(bool bio, int type, const ConvWs& w, const void* const* p, int64_t l, int64_t C, float* grads, const int64_t* o) {
  if (bio) return EdgeTerm{w.S, kBioQ, kBioQ, w.T + l * kBioQ * C, nullptr, 1, w.gT + l * kBioQ * C, nullptr, false};
  const int et = type == PGNN_CONV_GAT ? A_ET1 : G_ET1;
  return EdgeTerm{w.S, kChemQ, kChemQSplit, type == PGNN_CONV_GAT ? w.T + l * kChemQ * C : (const float*)p[et], (const float*)p[et + 1], 0,
                  grads ? grads + o[et] : nullptr, grads ? grads + o[et + 1] : nullptr, true};
}

// Every layer of a forward: Linear -> GAT | GCN gather | mean gather + L2 normalisation, then chem's BatchNorm (train or eval;
// its apply takes the ReLU and dropout) or bio's ReLU + dropout sweep.
int conv_forward(bool bio, int type, const void* const* params, const BnRun& bn, const void* edge_attr, int64_t N, int64_t E, int64_t L,
                 int64_t D, int training, const Drops& drops, int precision, float* node_rep, int64_t ld_out, const ConvWs& w,
                 cudaStream_t st) {
  const bool gat = type == PGNN_CONV_GAT;
  const int64_t C = gat ? kHeads * D : D;
  const int PL = bio ? bio_layer_params(type) : layer_params(type);
  const float* h = w.h0;
  for (int64_t l = 0; l < L; ++l) {
    const void* const* p = params + (bio ? PB_LAYER0 : P_LAYER0) + l * PL;
    const bool last = l == L - 1;
    const PgnnDropout drop = drops.at(l);
    const EdgeTerm e = edge_term(bio, type, w, p, l, C, nullptr, nullptr);
    float* xl = w.xl + l * N * C;
    float* z = w.z + l * N * D;
    // bio: the last layer without dropout writes node_rep itself, except GraphSAGE, whose backward reads its normalised rows from z
    const bool direct = bio && last && drop.p == 0.f && type != PGNN_CONV_SAGE && ld_out % 4 == 0 && aligned16(node_rep);
    float* out = direct ? node_rep : z;
    const int64_t ldo = direct ? ld_out : D;
    TRY(pgnn_linear_fwd(h, D, (const float*)p[CV_W], (const float*)p[CV_B], N, C, D, 0, xl, C, precision, st));
    if (gat) {
      if (!bio) {  // the kernels index one [9, H*D] table: rows 0..5 bond type, 6..8 bond direction
        float* T = w.T + l * kChemQ * C;
        PGNN_CUDA(cudaMemcpyAsync(T, p[A_ET1], sizeof(float) * 6 * C, cudaMemcpyDeviceToDevice, st));
        PGNN_CUDA(cudaMemcpyAsync(T + 6 * C, p[A_ET2], sizeof(float) * 3 * C, cudaMemcpyDeviceToDevice, st));
      }
      TRY(pgnn_gat_fwd(xl, N, kHeads, D, (const float*)p[CV_ATT], e.T, e.is_bio, edge_attr, w.rowptr_t, w.nbr_t, w.eid_t, E,
                       (const float*)p[CV_BIAS], kSlope, w.alpha + l * (E + N) * kHeads, w.pq + l * N * kHeads * 2, out, ldo, st));
    } else if (type == PGNN_CONV_GCN) {
      TRY(pgnn_internal_aggregate_fwd(xl, D, nullptr, nullptr, 0, N, D, w.rowptr_t, w.nbr_t, PGNN_AGG_GCN, w.dinv, e.S, e.Q, e.T, e.T2,
                                      e.q_split, 0, out, ldo, st, nullptr, nullptr));
    } else {
      // mean aggregation into the backward scratch `gz` (only its normalised rows and their norms are needed later)
      TRY(pgnn_internal_aggregate_fwd(xl, D, nullptr, nullptr, 0, N, D, w.rowptr_t, w.nbr_t, PGNN_AGG_MEAN, nullptr, e.S, e.Q, e.T, e.T2,
                                      e.q_split, 0, w.gz, D, st, nullptr, nullptr));
      TRY(pgnn_l2norm_fwd(w.gz, D, N, D, z, D, w.nrm + l * N, st));
    }
    float* hout = w.hout + l * N * D;
    if (bio) {
      if (!last) TRY(bio_act(false, z, D, nullptr, 0, N, D, 1, drop, hout, D, st));
      else if (!direct) TRY(bio_act(false, z, D, nullptr, 0, N, D, 0, drop, node_rep, ld_out, st));
    } else {
      if (last) hout = node_rep;
      const int64_t ldh = last ? ld_out : D;
      const float* gamma = (const float*)p[gat ? A_GAMMA : G_GAMMA];
      const float* beta = (const float*)p[gat ? A_BETA : G_BETA];
      if (training) {
        // after the ReLU: hout is the next layer's input and its Linear's weight-gradient operand
        TRY(pgnn_internal_bn_fwd_train(z, D, N, D, gamma, beta, bn.rm(l), bn.rv(l), bn.nb(l), bn.momentum, bn.eps, !last, hout, ldh,
                                       w.mean + l * D, w.invstd + l * D, nullptr, nullptr, w.scratch, w.scratch_bytes, st, &drop));
      } else {
        TRY(pgnn_bn_fwd_eval(z, D, N, D, gamma, beta, bn.rm(l), bn.rv(l), bn.eps, !last, hout, ldh, st));
      }
    }
    h = hout;
  }
  return PGNN_OK;
}

// Every layer of a backward: the gradient at the conv's output (chem: BatchNorm backward; bio: the ReLU + dropout sweep), then
// GAT backward | L2-normalisation backward + edge-table gradient + transpose gather, the Linear's weight gradient on the side
// stream and its input gradient.  x is chem's int64 atom codes or bio's float labels.
int conv_backward(bool bio, int type, const void* const* params, const float* g_node_rep, int64_t ldg, const void* x,
                  const void* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D, const Drops& drops, int precision, float* grads,
                  const int64_t* off, const ConvWs& w, cudaStream_t st) {
  const bool gat = type == PGNN_CONV_GAT;
  const int64_t C = gat ? kHeads * D : D;
  const int PL = bio ? bio_layer_params(type) : layer_params(type);
  const int layer0 = bio ? PB_LAYER0 : P_LAYER0;
  SideCtx* sc = precision == 1 ? side_ctx(st) : nullptr;
  if (bio && !gat) PGNN_CUDA(cudaMemsetAsync(w.gT, 0, sizeof(float) * L * kBioQ * C, st));
  const float* gy = g_node_rep;
  int64_t ldgy = ldg;
  for (int64_t l = L - 1; l >= 0; --l) {
    const void* const* p = params + layer0 + l * PL;
    const int64_t* o = off + layer0 + l * PL;
    const bool last = l == L - 1;
    const int par = (int)(l & 1);
    const float* xl = w.xl + l * N * C;
    const float* z = w.z + l * N * D;
    const float* hin = l == 0 ? w.h0 : w.hout + (l - 1) * N * D;
    float* gxl = w.gxl + (sc ? par * N * C : 0);
    const EdgeTerm e = edge_term(bio, type, w, p, l, C, grads, o);
    const PgnnDropout drop = drops.at(l);
    const float* gz = w.gz;
    int64_t ldgz = D;
    if (bio) {
      TRY(bio_act_bwd(gz, ldgz, gy, ldgy, z, N, D, last, drop, w.gz, st));
    } else {
      const int g = gat ? A_GAMMA : G_GAMMA, b = gat ? A_BETA : G_BETA;
      TRY(pgnn_internal_bn_bwd(gy, ldgy, z, D, N, D, (const float*)p[g], (const float*)p[b], w.mean + l * D, w.invstd + l * D, !last,
                               w.gz, D, grads + o[g], grads + o[b], nullptr, w.scratch, w.scratch_bytes, st, &drop));
    }
    TRY(side_wait(sc, st, 0, par));
    if (gat) {
      TRY(pgnn_gat_bwd(gz, ldgz, xl, N, kHeads, D, (const float*)p[CV_ATT], e.T, e.is_bio, edge_attr, w.rowptr_t, w.nbr_t, w.eid_t,
                       w.rowptr_s, w.nbr_s, w.eid_s, E, kSlope, w.alpha + l * (E + N) * kHeads, w.pq + l * N * kHeads * 2, gxl,
                       grads + o[CV_ATT], e.gT, grads + o[CV_BIAS], w.scratch, w.scratch_bytes, st));
    } else {
      const float* ga = gz;
      int64_t ldga = ldgz;
      if (type == PGNN_CONV_SAGE) {
        TRY(pgnn_l2norm_bwd(gz, ldgz, z, D, w.nrm + l * N, N, D, w.ga, D, st));
        ga = w.ga;
        ldga = D;
      }
      if (e.zero_gT) PGNN_CUDA(cudaMemsetAsync(e.gT, 0, sizeof(float) * e.Q * C, st));  // chem: the two tables are adjacent
      TRY(pgnn_internal_edge_table_bwd2(e.S, e.Q, ga, ldga, 0, N, (int)D, e.gT, D, e.gT2, e.q_split, st));
      TRY(pgnn_aggregate_bwd(ga, ldga, N, D, w.rowptr_s, w.nbr_s, agg_mode(type), w.dinv, w.rowptr_t, gxl, D, st));
    }
    // Linear: weight + bias gradients (side stream), then the input gradient
    TRY(side_wgrad(sc, st, 0, par, precision, gxl, C, hin, D, N, C, D, grads + o[CV_W], grads + o[CV_B], w.wpart, w.wpart_floats));
    TRY(pgnn_linear_bwd_x(gxl, C, (const float*)p[CV_W], N, C, D, nullptr, 0, w.gh, D, precision, st));
    gy = w.gh;
    ldgy = D;
  }
  if (bio) return bio_backward_tail(type, sc, w.gT, w.gh, (const float*)x, N, L, D, grads, off, st);
  return embed_backward(sc, w, w.gh, (const int64_t*)x, N, D, precision, grads, off, w.wpart, w.wpart_floats, st);
}

int64_t workspace_bytes(bool bio, int type, int64_t N, int64_t E, int64_t L, int64_t D) {
  if (type != kGin) return carve_conv(nullptr, bio, type, N, E, L, D).total;
  return bio ? carve_bio_gin(nullptr, N, E, L, D).total : carve_gin(nullptr, N, E, L, D).total;
}

// The start of every pass of either domain, in this order: the checks both passes share plus `ok` (the pass's own), the
// workspace size, then N == 0, which ends the call (run = false; a backward zeroes its gradients).  A backward (off != nullptr)
// gets its flat gradient layout.
int begin_pass(bool bio, int type, float drop_p, bool ok, int64_t N, int64_t E, int64_t L, int64_t D, const void* params,
               void* workspace, int64_t workspace_size, float* grads, std::vector<int64_t>* off, cudaStream_t st, bool& run) {
  run = false;
  PGNN_CHECK_ARG(valid_type(type) && drop_p >= 0.f && drop_p <= 1.f && ok);
  PGNN_CHECK_ARG(N >= 0 && E >= 0 && L >= 1 && D > 0 && D % 4 == 0 && params && workspace);
  if (workspace_size < workspace_bytes(bio, type, N, E, L, D)) return PGNN_EWORKSPACE;
  if (off) {
    off->resize((bio ? bio_grad_layout(type, L, D, nullptr) : grad_layout(type, L, D, nullptr)) + 1);
    if (bio) bio_grad_layout(type, L, D, off->data());
    else grad_layout(type, L, D, off->data());
  }
  if (N == 0) {
    if (off) PGNN_CUDA(cudaMemsetAsync(grads, 0, sizeof(float) * off->back(), st));
    return PGNN_OK;
  }
  run = true;
  return PGNN_OK;
}

}  // namespace

extern "C" {

// ------------------------------------------------------------------------------------------------------------------------------
// GIN
// ------------------------------------------------------------------------------------------------------------------------------
int64_t pgnn_chem_gin_num_params(int64_t L) { return L < 1 ? PGNN_EINVAL : grad_layout(kGin, L, 0, nullptr); }

int pgnn_chem_gin_grad_offsets(int64_t L, int64_t D, int64_t* offsets /*host [num_params + 1]*/) {
  PGNN_CHECK_ARG(L >= 1 && D > 0 && offsets);
  grad_layout(kGin, L, D, offsets);
  return PGNN_OK;
}

int64_t pgnn_chem_gin_workspace_bytes(int64_t N, int64_t E, int64_t L, int64_t D) {
  if (N < 0 || E < 0 || L < 1 || D <= 0) return PGNN_EINVAL;
  return workspace_bytes(false, kGin, N, E, L, D);
}

int pgnn_chem_gin_forward(const void* const* params, void* const* bn_running_mean, void* const* bn_running_var,
                          void* const* bn_num_batches_tracked, const int64_t* x, const int64_t* edge_index,
                          const int64_t* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D, int training, float momentum, float eps,
                          int precision, float* node_rep, int64_t ld_out, void* workspace, int64_t workspace_bytes, void* stream) {
  return pgnn_chem_encoder_forward(kGin, params, bn_running_mean, bn_running_var, bn_num_batches_tracked, x, edge_index, edge_attr, N, E, L, D,
                                   training, momentum, eps, 0.f, 0, precision, node_rep, ld_out, workspace, workspace_bytes, stream);
}

int pgnn_chem_gin_backward(const void* const* params, const float* g_node_rep, int64_t ldg, const int64_t* x, int64_t N, int64_t E,
                           int64_t L, int64_t D, int precision, float* grads, void* workspace, int64_t workspace_bytes,
                           void* stream) {
  return pgnn_chem_encoder_backward(kGin, params, g_node_rep, ldg, x, nullptr, N, E, L, D, 0.f, 0, precision, grads, workspace,
                                    workspace_bytes, stream);
}

// Development / test aid: byte offsets inside the workspace of the saved activations a test needs to reconstruct the
// ReLU decisions the encoder actually took: out[0] = z1 (post-ReLU hidden activations, [L][N][2D]), out[1] = z2 (pre-BatchNorm
// layer outputs, [L][N][D]), out[2] = BatchNorm batch mean [L][D], out[3] = invstd [L][D].
int pgnn_chem_gin_debug_layout(int64_t N, int64_t E, int64_t L, int64_t D, int64_t* out4) {
  PGNN_CHECK_ARG(N >= 0 && E >= 0 && L >= 1 && D > 0 && out4);
  char* base = reinterpret_cast<char*>(0x1000);  // carve_gin() only does pointer arithmetic
  GinWs w = carve_gin(base, N, E, L, D);
  out4[0] = reinterpret_cast<char*>(w.z1) - base;
  out4[1] = reinterpret_cast<char*>(w.z2) - base;
  out4[2] = reinterpret_cast<char*>(w.mean) - base;
  out4[3] = reinterpret_cast<char*>(w.invstd) - base;
  return PGNN_OK;
}

// Test aid: byte offset inside the workspace of aggr ([L][N][D]): layer l's gathered input, i.e. for l > 0 the previous layer's
// BatchNorm + ReLU as the gather applied it on load (with no edges and zero edge tables, exactly act(z2[l-1]) row for row)
int64_t pgnn_chem_gin_debug_aggr_offset(int64_t N, int64_t E, int64_t L, int64_t D) {
  if (N < 0 || E < 0 || L < 1 || D <= 0) return PGNN_EINVAL;
  char* base = reinterpret_cast<char*>(0x1000);
  GinWs w = carve_gin(base, N, E, L, D);
  return reinterpret_cast<char*>(w.aggr) - base;
}

// ------------------------------------------------------------------------------------------------------------------------------
// GCN / GraphSAGE / GAT
// ------------------------------------------------------------------------------------------------------------------------------
int64_t pgnn_chem_conv_num_params(int conv_type, int64_t L) {
  if (!valid_conv(conv_type) || L < 1) return PGNN_EINVAL;
  return grad_layout(conv_type, L, 0, nullptr);
}

int pgnn_chem_conv_grad_offsets(int conv_type, int64_t L, int64_t D, int64_t* offsets) {
  PGNN_CHECK_ARG(valid_conv(conv_type) && L >= 1 && D > 0 && offsets);
  grad_layout(conv_type, L, D, offsets);
  return PGNN_OK;
}

int64_t pgnn_chem_conv_workspace_bytes(int conv_type, int64_t N, int64_t E, int64_t L, int64_t D) {
  if (!valid_conv(conv_type) || N < 0 || E < 0 || L < 1 || D <= 0) return PGNN_EINVAL;
  return workspace_bytes(false, conv_type, N, E, L, D);
}

int pgnn_chem_conv_forward(int conv_type, const void* const* params, void* const* bn_running_mean, void* const* bn_running_var,
                           void* const* bn_num_batches_tracked, const int64_t* x, const int64_t* edge_index, const int64_t* edge_attr,
                           int64_t N, int64_t E, int64_t L, int64_t D, int training, float momentum, float eps, int precision,
                           float* node_rep, int64_t ld_out, void* workspace, int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(valid_conv(conv_type));
  return pgnn_chem_encoder_forward(conv_type, params, bn_running_mean, bn_running_var, bn_num_batches_tracked, x, edge_index, edge_attr, N, E, L,
                                   D, training, momentum, eps, 0.f, 0, precision, node_rep, ld_out, workspace, workspace_bytes, stream);
}

int pgnn_chem_conv_backward(int conv_type, const void* const* params, const float* g_node_rep, int64_t ldg, const int64_t* x,
                            const int64_t* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D, int precision, float* grads,
                            void* workspace, int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(valid_conv(conv_type));
  return pgnn_chem_encoder_backward(conv_type, params, g_node_rep, ldg, x, edge_attr, N, E, L, D, 0.f, 0, precision, grads, workspace,
                                    workspace_bytes, stream);
}

// ------------------------------------------------------------------------------------------------------------------------------
// every type, with dropout
// ------------------------------------------------------------------------------------------------------------------------------
int pgnn_chem_encoder_forward(int gnn_type, const void* const* params, void* const* bn_running_mean, void* const* bn_running_var,
                              void* const* bn_num_batches_tracked, const int64_t* x, const int64_t* edge_index, const int64_t* edge_attr,
                              int64_t N, int64_t E, int64_t L, int64_t D, int training, float momentum, float eps, float drop_p,
                              int64_t drop_seed, int precision, float* node_rep, int64_t ld_out, void* workspace, int64_t workspace_bytes,
                              void* stream) {
  cudaStream_t st = as_stream(stream);
  bool run;
  TRY(begin_pass(false, gnn_type, drop_p,
                 bn_running_mean && bn_running_var && (N == 0 || (x && node_rep)) && (gnn_type == kGin || E == 0 || (edge_index && edge_attr)),
                 N, E, L, D, params, workspace, workspace_bytes, nullptr, nullptr, st, run));
  if (!run) return PGNN_OK;
  Drops drops;
  if (training) drops = Drops{drop_p, drop_seed};  // eval mode has no dropout
  const BnRun bn{bn_running_mean, bn_running_var, bn_num_batches_tracked, momentum, eps};
  if (gnn_type == kGin) {
    const GinWs w = carve_gin(workspace, N, E, L, D);
    TRY(forward_prologue(kGin, w, params, x, edge_index, edge_attr, N, E, D, training, precision, w.scratch, w.scratch_bytes, st));
    return gin_forward(params, bn, training, drops, precision, node_rep, ld_out, N, L, D, w, st);
  }
  const ConvWs w = carve_conv(workspace, false, gnn_type, N, E, L, D);
  TRY(forward_prologue(gnn_type, w, params, x, edge_index, edge_attr, N, E, D, training, precision, w.scratch, w.scratch_bytes, st));
  return conv_forward(false, gnn_type, params, bn, edge_attr, N, E, L, D, training, drops, precision, node_rep, ld_out, w, st);
}

int pgnn_chem_encoder_backward(int gnn_type, const void* const* params, const float* g_node_rep, int64_t ldg, const int64_t* x,
                               const int64_t* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D, float drop_p, int64_t drop_seed,
                               int precision, float* grads, void* workspace, int64_t workspace_bytes, void* stream) {
  cudaStream_t st = as_stream(stream);
  std::vector<int64_t> off;
  bool run;
  TRY(begin_pass(false, gnn_type, drop_p, grads != nullptr, N, E, L, D, params, workspace, workspace_bytes, grads, &off, st, run));
  if (!run) return PGNN_OK;
  PGNN_CHECK_ARG(g_node_rep && x && (gnn_type == kGin || E == 0 || edge_attr));
  const Drops drops{drop_p, drop_seed};
  if (gnn_type == kGin)
    return gin_backward(params, g_node_rep, ldg, x, N, L, D, drops, precision, grads, off.data(), carve_gin(workspace, N, E, L, D), st);
  return conv_backward(false, gnn_type, params, g_node_rep, ldg, x, edge_attr, N, E, L, D, drops, precision, grads, off.data(),
                       carve_conv(workspace, false, gnn_type, N, E, L, D), st);
}

// ------------------------------------------------------------------------------------------------------------------------------
// bio, every type, with dropout
// ------------------------------------------------------------------------------------------------------------------------------
int64_t pgnn_bio_encoder_num_params(int gnn_type, int64_t L) {
  if (!valid_type(gnn_type) || L < 1) return PGNN_EINVAL;
  return bio_grad_layout(gnn_type, L, 0, nullptr);
}

int pgnn_bio_encoder_grad_offsets(int gnn_type, int64_t L, int64_t D, int64_t* offsets) {
  PGNN_CHECK_ARG(valid_type(gnn_type) && L >= 1 && D > 0 && offsets);
  bio_grad_layout(gnn_type, L, D, offsets);
  return PGNN_OK;
}

int64_t pgnn_bio_encoder_workspace_bytes(int gnn_type, int64_t N, int64_t E, int64_t L, int64_t D) {
  if (!valid_type(gnn_type) || N < 0 || E < 0 || L < 1 || D <= 0) return PGNN_EINVAL;
  return workspace_bytes(true, gnn_type, N, E, L, D);
}

int pgnn_bio_encoder_forward(int gnn_type, const void* const* params, void* const* bn_running_mean, void* const* bn_running_var,
                             void* const* bn_num_batches_tracked, const float* x, const int64_t* edge_index, const float* edge_attr,
                             int64_t N, int64_t E, int64_t L, int64_t D, int training, float momentum, float eps, float drop_p,
                             int64_t drop_seed, int precision, float* node_rep, int64_t ld_out, void* workspace, int64_t workspace_bytes,
                             void* stream) {
  cudaStream_t st = as_stream(stream);
  bool run;
  TRY(begin_pass(true, gnn_type, drop_p,
                 (gnn_type != kGin || (bn_running_mean && bn_running_var)) && (N == 0 || (x && node_rep && ld_out >= D)) &&
                     (E == 0 || (edge_index && edge_attr)),
                 N, E, L, D, params, workspace, workspace_bytes, nullptr, nullptr, st, run));
  if (!run) return PGNN_OK;
  Drops drops;
  if (training) drops = Drops{drop_p, drop_seed};  // eval mode has no dropout
  const BnRun bn{bn_running_mean, bn_running_var, bn_num_batches_tracked, momentum, eps};
  if (gnn_type == kGin) {
    const BioGinWs w = carve_bio_gin(workspace, N, E, L, D);
    TRY(bio_prologue(kGin, w, w.T, params, x, edge_index, edge_attr, N, E, L, D, w.scratch, w.scratch_bytes, st));
    return bio_gin_forward(params, bn, N, L, D, training, drops, precision, node_rep, ld_out, w, st);
  }
  const ConvWs w = carve_conv(workspace, true, gnn_type, N, E, L, D);
  TRY(bio_prologue(gnn_type, w, w.T, params, x, edge_index, edge_attr, N, E, L, D, w.scratch, w.scratch_bytes, st));
  return conv_forward(true, gnn_type, params, bn, edge_attr, N, E, L, D, training, drops, precision, node_rep, ld_out, w, st);
}

int pgnn_bio_encoder_backward(int gnn_type, const void* const* params, const float* g_node_rep, int64_t ldg, const float* x,
                              const float* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D, float drop_p, int64_t drop_seed,
                              int precision, float* grads, void* workspace, int64_t workspace_bytes, void* stream) {
  cudaStream_t st = as_stream(stream);
  std::vector<int64_t> off;
  bool run;
  TRY(begin_pass(true, gnn_type, drop_p, grads != nullptr, N, E, L, D, params, workspace, workspace_bytes, grads, &off, st, run));
  if (!run) return PGNN_OK;
  PGNN_CHECK_ARG(g_node_rep && x && ldg >= D && (E == 0 || gnn_type != PGNN_CONV_GAT || edge_attr));
  const Drops drops{drop_p, drop_seed};
  if (gnn_type == kGin)
    return bio_gin_backward(params, g_node_rep, ldg, x, N, L, D, drops, precision, grads, off.data(), carve_bio_gin(workspace, N, E, L, D),
                            st);
  return conv_backward(true, gnn_type, params, g_node_rep, ldg, x, edge_attr, N, E, L, D, drops, precision, grads, off.data(),
                       carve_conv(workspace, true, gnn_type, N, E, L, D), st);
}

}  // extern "C"
