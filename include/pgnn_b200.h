/*
 * pgnn_b200.h — C ABI of libpgnn_b200.so: the H100 (sm_90a) message-passing hot path of
 * snap-stanford/pretrain-gnns (chem/model.py, bio/model.py).
 *
 * The reference exposes NO native interface for this path: its arithmetic runs inside
 * torch_geometric 1.0.3 / torch_scatter 1.1.2 / ATen (requirements.txt:2-7).  These entry points are
 * what a binding for the path has to call; each one cites the reference lines it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless it says "host"; row-major; fp32 unless noted
 *   - `ld*` are row strides in ELEMENTS
 *   - edge_index[0] is the aggregation TARGET, edge_index[1] the SOURCE (PyG 1.0.x flow)
 *   - self-loops are implicit: every node has one, ordered after its real in-edges (chem/model.py:39)
 *   - `stream` is a cudaStream_t passed as void*; calls only enqueue work (no host sync), keep no
 *     references to caller memory after the enqueued work completes, and are re-entrant per stream
 *   - return 0 on success, a negative PGNN_E* code otherwise; nothing throws across the boundary
 */
#ifndef PGNN_B200_H
#define PGNN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PGNN_API __attribute__((visibility("default")))

#define PGNN_OK 0
#define PGNN_EINVAL (-1)      /* bad argument (null pointer, negative size, unsupported width) */
#define PGNN_ECUDA (-2)       /* a CUDA call / launch failed; see pgnn_last_cuda_error() */
#define PGNN_EWORKSPACE (-3)  /* workspace smaller than the *_workspace_bytes query */
#define PGNN_EUNSUPPORTED (-4)

/* Index preconditions.  Every index the kernels consume must be in range: node ids of edge_index and segment ids in
 * [0, num_nodes / num_segments), atom codes in [0,120) x [0,3) (chem/model.py:9-10), bond codes in [0,6) x [0,3) (:12-13),
 * class labels in [0, V), gather indices in [0, rows).  The reference's torch ops raise a device-side assert otherwise; here
 * the consuming kernel drops / clamps the offending element (never reads or writes out of range) and ORs one of these bits
 * into a per-device error word, which pgnn_device_error_flags() reads back (it synchronises the device). */
#define PGNN_DEVERR_NODE_ID 1u     /* edge_index entry or segment id (graph_prep, bucket) */
#define PGNN_DEVERR_ATOM_CODE 2u   /* chem x[:,0] / x[:,1] (chem_embed_*, chem_gin_*) */
#define PGNN_DEVERR_BOND_CODE 4u   /* chem edge_attr (chem_edge_summary, gat) */
#define PGNN_DEVERR_LABEL 8u       /* softmax_ce labels */
#define PGNN_DEVERR_GATHER 16u     /* row_gather indices */

/* reduction modes of the neighbour aggregation */
#define PGNN_AGG_SUM 0   /* GIN:  chem/model.py:49,  bio/model.py:52            */
#define PGNN_AGG_MEAN 1  /* SAGE: chem/model.py:169, bio/model.py:184 (count = in-degree + 1) */
#define PGNN_AGG_GCN 2   /* GCN:  chem/model.py:73-82,103-104  w = deg^-1/2[t] * deg^-1/2[s] */

PGNN_API int pgnn_version(void);
PGNN_API const char* pgnn_error_string(int code);
PGNN_API int pgnn_last_cuda_error(void);
/* Synchronise the current device and return its PGNN_DEVERR_* bits (>= 0; negative = error code); clear != 0 resets them. */
PGNN_API int pgnn_device_error_flags(int clear);          /* cudaError_t of the last PGNN_ECUDA on this thread */
PGNN_API int pgnn_device_sm_count(int device);   /* host query; negative on error */
PGNN_API int64_t pgnn_kernel_launch_count(void); /* kernels this library has enqueued since load (process-wide) */
/* Per-kernel timing mode: while enabled, every kernel launch of the library is bracketed by a CUDA event pair on its own
 * stream (this serialises neighbouring kernels: use it for a few diagnostic steps, not for the number you report).
 * pgnn_profile_read waits for the recorded events, writes "kernel name<TAB>launches<TAB>total_us" lines into buf
 * (host memory, NUL-terminated, truncated to buflen), clears the records and returns the number of launches covered. */
PGNN_API int pgnn_profile_enable(int on);
PGNN_API int64_t pgnn_profile_read(char* buf, int64_t buflen);

/* ---------------------------------------------------------------------------------------------
 * Graph preparation (integer, bit-exact).  Replaces the per-layer, per-edge gather / scatter_add
 * addressing done by MessagePassing.propagate (chem/model.py:49 [PyG 1.0.3]) with one bucketing per
 * batch that all layers and both passes reuse.
 * ------------------------------------------------------------------------------------------- */

/* Stable counting sort of `num_keys` int64 keys (stride `key_stride` elements) into `num_buckets`
 * buckets.  rowptr[num_buckets+1]; order[num_keys] = original positions, bucket by bucket, ascending
 * inside a bucket.  If vals != NULL (int64, stride val_stride), vals_out[p] = (int32) vals[order[p]].
 * Keys outside [0, num_buckets) are undefined behaviour, as in the reference. */
PGNN_API int64_t pgnn_bucket_workspace_bytes(int64_t num_keys, int64_t num_buckets);
PGNN_API int pgnn_bucket(const int64_t* keys, int64_t key_stride, int64_t num_keys, int64_t num_buckets,
                         const int64_t* vals, int64_t val_stride,
                         int32_t* rowptr, int32_t* order, int32_t* vals_out,
                         void* workspace, int64_t workspace_bytes, void* stream);

/* edge_index int64 [2,E] -> by-target CSR (rowptr_t[N+1], nbr_t[E] = sources, eid_t[E]) and
 * by-source CSR (rowptr_s, nbr_s = targets, eid_s).  Two pgnn_bucket passes. */
PGNN_API int64_t pgnn_graph_prep_workspace_bytes(int64_t num_nodes, int64_t num_edges);
PGNN_API int pgnn_graph_prep(const int64_t* edge_index, int64_t num_edges, int64_t num_nodes,
                             int32_t* rowptr_t, int32_t* nbr_t, int32_t* eid_t,
                             int32_t* rowptr_s, int32_t* nbr_s, int32_t* eid_s,
                             void* workspace, int64_t workspace_bytes, void* stream);

/* dinv[i] = (in_degree(i) + 1)^-1/2  (GCN norm, chem/model.py:75-80; the +1 is the self-loop) */
PGNN_API int pgnn_gcn_dinv(const int32_t* rowptr_t, int64_t num_nodes, float* dinv, void* stream);

/* Per-node edge-feature summary S[N,Q]: because the message is LINEAR in the edge embedding, the
 * per-edge embedding rows of chem/model.py:47 / bio/model.py:47 are never materialised:
 *   sum_k w_k * e_k  =  S[i,:] . T      with T the [Q,C] table / transposed encoder (see aggregate).
 * chem (Q = 9):  S[i,a] += w_k for bond type a = edge_attr[k,0] in 0..5, S[i,6+d] += w_k for direction d;
 *                self-loop counts as type 4, direction 0 (chem/model.py:42-45).
 * bio  (Q = 10): S[i,0:9] += w_k * edge_attr[k,0:9], self-loop adds w_ii to column 7 (bio/model.py:42-43);
 *                S[i,9] = sum of weights (multiplies the encoder bias).
 * w_k by `mode` (PGNN_AGG_*; dinv required for GCN). */
PGNN_API int pgnn_chem_edge_summary(const int64_t* edge_attr /*[E,2]*/, const int32_t* rowptr_t,
                                    const int32_t* nbr_t, const int32_t* eid_t, int64_t num_nodes,
                                    int mode, const float* dinv, float* S /*[N,9]*/, void* stream);
PGNN_API int pgnn_bio_edge_summary(const float* edge_attr /*[E,9]*/, const int32_t* rowptr_t,
                                   const int32_t* nbr_t, const int32_t* eid_t, int64_t num_nodes,
                                   int mode, const float* dinv, float* S /*[N,10]*/, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Input embeddings.  chem/model.py:264  h0 = E1[x[:,0]] + E2[x[:,1]];  bio/model.py:49-50
 * h0 = E[(long) x] (one table, float-coded index).
 * ------------------------------------------------------------------------------------------- */
PGNN_API int pgnn_chem_embed_fwd(const int64_t* x /*[N,2]*/, const float* tab1, int64_t rows1, const float* tab2, int64_t rows2,
                                 int64_t num_nodes, int64_t C, float* out, int64_t ldo, void* stream);
/* gtab1 [rows1,C], gtab2 [rows2,C] are OVERWRITTEN (zeroed, then accumulated) */
PGNN_API int pgnn_chem_embed_bwd(const int64_t* x, const float* g, int64_t ldg, int64_t num_nodes, int64_t C,
                                 float* gtab1, int64_t rows1, float* gtab2, int64_t rows2, void* stream);
PGNN_API int pgnn_bio_embed_fwd(const float* x /*[N]*/, const float* tab /*[2,C]*/, int64_t num_nodes,
                                int64_t C, float* out, int64_t ldo, void* stream);
PGNN_API int pgnn_bio_embed_bwd(const float* x, const float* g, int64_t ldg, int64_t num_nodes, int64_t C,
                                float* gtab /*[2,C]*/, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Neighbour aggregation (the gather + scatter_add of propagate, chem/model.py:49,101,196 and
 * bio/model.py:52,111,218), atomics-free: one thread group per target row walks its bucket in edge
 * order, self-loop last.
 *
 *   out[i, 0:C]           = sum_k w_k * x[nbr_t[k], 0:C] + w_ii * x[i, 0:C]   (+ S[i,:] . T if edge_off == 0)
 *   out[i, edge_off: +C]  = S[i,:] . T                                       (if edge_off > 0: bio GIN concat,
 *                                                                              bio/model.py:54-55)
 * x may be given as (pre-BN activations, per-column affine, ReLU flag): x_eff = act(fmaf(x, in_scale, in_shift))
 * so a BatchNorm + ReLU (chem/model.py:269-275) is applied on load instead of in a pass of its own
 * (in_scale == NULL -> identity).  The ReLU keeps NaN, as torch.relu does.
 * ------------------------------------------------------------------------------------------- */
PGNN_API int pgnn_aggregate_fwd(const float* x, int64_t ldx, const float* in_scale, const float* in_shift,
                                int in_relu, int64_t num_nodes, int64_t C,
                                const int32_t* rowptr_t, const int32_t* nbr_t, int mode, const float* dinv,
                                const float* S, int64_t Q, const float* T /*[Q,C]*/, int64_t edge_off,
                                float* out, int64_t ldo, void* stream);
/* gx[j,0:C] = sum_{k: src_k = j} w_k * g[tgt_k, 0:C] + w_jj * g[j, 0:C]     (transpose-graph gather) */
PGNN_API int pgnn_aggregate_bwd(const float* g, int64_t ldg, int64_t num_nodes, int64_t C,
                                const int32_t* rowptr_s, const int32_t* nbr_s, int mode, const float* dinv,
                                const int32_t* rowptr_t, float* gx, int64_t ldgx, void* stream);
/* gT[Q,C] = S^T . g[:, g_off : g_off+C]   (edge-table / edge-encoder gradient; gT OVERWRITTEN) */
PGNN_API int pgnn_edge_table_bwd(const float* S, int64_t Q, const float* g, int64_t ldg, int64_t g_off,
                                 int64_t num_nodes, int64_t C, float* gT, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Dense node transforms (torch.nn.Linear inside GINConv.mlp chem/model.py:29, bio/model.py:24;
 * GCN/SAGE/GAT linear chem/model.py:99,147,194).  precision: 0 = fp32 FFMA (SIMT),
 * 1 = 3xTF32 error-compensated wgmma (falls back to 0 where a shape is unsupported).
 * ------------------------------------------------------------------------------------------- */
/* y[M,N] = act(x[M,K] . w[N,K]^T + bias[N]) ; relu != 0 applies max(.,0) */
PGNN_API int pgnn_linear_fwd(const float* x, int64_t ldx, const float* w, const float* bias,
                             int64_t M, int64_t N, int64_t K, int relu, float* y, int64_t ldy,
                             int precision, void* stream);
/* gx[M,K] = (gy[M,N] . w[N,K]) * (relu_src > 0 ? 1 : 0)   relu_src: [M,K] activations or NULL */
PGNN_API int pgnn_linear_bwd_x(const float* gy, int64_t ldgy, const float* w, int64_t M, int64_t N, int64_t K,
                               const float* relu_src, int64_t ldr, float* gx, int64_t ldgx,
                               int precision, void* stream);
/* gw[N,K] = gy[M,N]^T . x[M,K] ; gb[N] = column sums of gy (gb may be NULL).  Outputs OVERWRITTEN. */
PGNN_API int pgnn_linear_bwd_w(const float* gy, int64_t ldgy, const float* x, int64_t ldx,
                               int64_t M, int64_t N, int64_t K, float* gw, float* gb,
                               int precision, void* stream);

/* ---------------------------------------------------------------------------------------------
 * BatchNorm1d (chem/model.py:252,269; bio/model.py:24), eps 1e-5, momentum 0.1 passed explicitly.
 * Statistics are accumulated in fp64 (block partials folded with fp64 atomics: order effects ~1e-16).
 * ------------------------------------------------------------------------------------------- */
PGNN_API int64_t pgnn_bn_workspace_bytes(int64_t M, int64_t C);
/* train: batch statistics (biased var), y = act(fmaf(x, scale, shift)) with scale = gamma*invstd and
 * shift = fmaf(-mean, scale, beta) (fp32, one rounding each); save_mean/save_invstd [C] written for backward;
 * running_mean/var (unbiased var) and *num_batches_tracked updated in place when non-NULL.  y may be NULL
 * (statistics only: the consumer applies scale/shift on load); scale/shift [C] are written when non-NULL.
 * Any 0 < M < 2^31. */
PGNN_API int pgnn_bn_fwd_train(const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma,
                               const float* beta, float* running_mean, float* running_var,
                               int64_t* num_batches_tracked, float momentum, float eps, int relu,
                               float* y, int64_t ldy, float* save_mean, float* save_invstd,
                               float* scale, float* shift, void* workspace, int64_t workspace_bytes,
                               void* stream);
PGNN_API int pgnn_bn_fwd_eval(const float* x, int64_t ldx, int64_t M, int64_t C, const float* gamma,
                              const float* beta, const float* running_mean, const float* running_var,
                              float eps, int relu, float* y, int64_t ldy, void* stream);
/* gx = BN'(gy * relu_mask); ggamma/gbeta [C] OVERWRITTEN.  relu != 0: mask = (y > 0) with y recomputed
 * bit for bit from x, save_mean, save_invstd, gamma, beta by the forward's expression above. */
PGNN_API int pgnn_bn_bwd(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t C,
                         const float* gamma, const float* beta, const float* save_mean,
                         const float* save_invstd, int relu, float* gx, int64_t ldgx, float* ggamma,
                         float* gbeta, void* workspace, int64_t workspace_bytes, void* stream);
/* y = relu(x), gx = gy * (y > 0): the inter-layer ReLU of bio/model.py:281 (no BatchNorm there).  relu keeps NaN, as
 * torch.relu does, here and in the BatchNorm entry points above. */
PGNN_API int pgnn_relu_fwd(const float* x, int64_t ldx, int64_t M, int64_t C, float* y, int64_t ldy, void* stream);
PGNN_API int pgnn_relu_bwd(const float* gy, int64_t ldgy, const float* y, int64_t ldy_, int64_t M, int64_t C,
                           float* gx, int64_t ldgx, void* stream);
/* Dropout (chem/model.py:271-275, bio/model.py:283-286: F.dropout(h, p, training=True)) with a DEFINED draw: element (row i,
 * column c) of layer `layer`'s [M, C] activation is kept iff
 *     r = splitmix64(seed, ((uint64)layer << 40) | (uint64)(i * C + c)) >> 32   (a uint32; splitmix64 as in pgnn_mask_atoms)
 *     r >= thr,   thr = floor(p * 2^32) for 0 <= p < 1;  p == 1 drops everything
 * and y = x * (kept ? scale : 0.f) with scale = (float)(1.0 / (1.0 - p)) (p as the float passed here).  A dropped NaN stays NaN and
 * a dropped +-Inf becomes NaN, as torch's x * mask * scale does.  The mask is a pure function of (seed, layer, i, c): the backward
 * gx = gy * (kept ? scale : 0.f) regenerates it, and no mask tensor exists.  torch's Philox stream cannot be matched, so the draw
 * is defined here (as for pgnn_mask_atoms); the distribution is the same.  0 <= layer < 2^24, M * C < 2^40; p outside [0, 1] or
 * NaN is PGNN_EINVAL. */
PGNN_API int pgnn_dropout_fwd(const float* x, int64_t ldx, int64_t M, int64_t C, float p, int64_t seed, int64_t layer, float* y,
                              int64_t ldy, void* stream);
PGNN_API int pgnn_dropout_bwd(const float* gy, int64_t ldgy, int64_t M, int64_t C, float p, int64_t seed, int64_t layer, float* gx,
                              int64_t ldgx, void* stream);
/* GraphSAGE update: y = x / max(||x||_2, 1e-12) per row (chem/model.py:201-202) and its backward */
PGNN_API int pgnn_l2norm_fwd(const float* x, int64_t ldx, int64_t M, int64_t C, float* y, int64_t ldy,
                             float* norm /*[M]*/, void* stream);
PGNN_API int pgnn_l2norm_bwd(const float* gy, int64_t ldgy, const float* y, int64_t ldy_, const float* norm,
                             int64_t M, int64_t C, float* gx, int64_t ldgx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * GAT (chem/model.py:134-165, bio/model.py:147-180), heads fixed by the caller (reference: 2).
 * xl [N,H*D] is weight_linear(x).  Edge embedding rows e_k [H*D] are  Tsel = T rows selected/combined
 * by the per-edge features: chem e_k = T[a0_k] + T[6 + a1_k] (T [9,H*D]); bio e_k = sum_q attr[k,q] T[q] +
 * T[9] (T [10,H*D] = [W^T ; b]).  `feat` is the raw edge_attr (int64 [E,2] for chem, float [E,9] for bio).
 * alpha [E+N, H] (target-bucket order, then the self-loop of node i at E+i) and pq [N,H,2] (the per-node
 * halves <att_i, xl_n> and <att_j, xl_n> of the attention logit) are written for backward.  D <= 320.
 * ------------------------------------------------------------------------------------------- */
PGNN_API int pgnn_gat_fwd(const float* xl, int64_t num_nodes, int64_t H, int64_t D, const float* att /*[H,2D]*/,
                          const float* T, int is_bio, const void* feat, const int32_t* rowptr_t,
                          const int32_t* nbr_t, const int32_t* eid_t, int64_t num_edges, const float* bias /*[D]*/,
                          float slope, float* alpha, float* pq, float* out /*[N,D]*/, int64_t ldo, void* stream);
PGNN_API int64_t pgnn_gat_bwd_workspace_bytes(int64_t num_nodes, int64_t num_edges, int64_t H, int64_t D);
/* gxl [N,H*D], gatt [H,2D], gT [Q,H*D] (Q = 9 chem / 10 bio), gbias [D]: all OVERWRITTEN */
PGNN_API int pgnn_gat_bwd(const float* g /*[N,D]*/, int64_t ldg, const float* xl, int64_t num_nodes, int64_t H,
                          int64_t D, const float* att, const float* T, int is_bio, const void* feat,
                          const int32_t* rowptr_t, const int32_t* nbr_t, const int32_t* eid_t,
                          const int32_t* rowptr_s, const int32_t* nbr_s, const int32_t* eid_s,
                          int64_t num_edges, float slope, const float* alpha, const float* pq,
                          float* gxl, float* gatt, float* gT, float* gbias,
                          void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Heads (chem/model.py:326,369; chem/pretrain_masking.py:51,58-59; chem/pretrain_contextpred.py:54-67;
 * bio/model.py:342-345).
 * ------------------------------------------------------------------------------------------- */
/* out[b,:] = mean of x rows whose segment id is b; `seg_ptr[B+1]`/`seg_order[N]` from pgnn_bucket(batch).
 * Empty segments give 0 (count.clamp(min=1)). */
PGNN_API int pgnn_segment_mean_fwd(const float* x, int64_t ldx, const int32_t* seg_ptr, const int32_t* seg_order,
                                   int64_t num_seg, int64_t C, float* out, int64_t ldo, void* stream);
/* gx[n,:] = g[seg[n],:] / max(count[seg[n]],1) ; seg = int64 ids [N] */
PGNN_API int pgnn_segment_mean_bwd(const float* g, int64_t ldg, const int64_t* seg, const int32_t* seg_ptr,
                                   int64_t num_rows, int64_t C, float* gx, int64_t ldgx, void* stream);
/* out[m,:] = x[idx[m],:] (+ x[idx2[m],:] if idx2 != NULL: the bond representation rep[u]+rep[v]) */
PGNN_API int pgnn_row_gather_fwd(const float* x, int64_t ldx, int64_t num_rows, const int64_t* idx, const int64_t* idx2,
                                 int64_t num_idx, int64_t C, float* out, int64_t ldo, void* stream);
/* gx[idx[m],:] += g[m,:] (and idx2). gx must be pre-initialised by the caller (accumulates). */
PGNN_API int pgnn_row_gather_bwd(const float* g, int64_t ldg, const int64_t* idx, const int64_t* idx2,
                                 int64_t num_idx, int64_t C, float* gx, int64_t ldgx, int64_t num_rows, void* stream);
/* Mean cross-entropy of fp32 logits [M,V] evaluated in fp64 (criterion(pred.double(), labels), chem/pretrain_masking.py:52).
 * *loss_mean (device fp64 scalar) is OVERWRITTEN; dlogits [M, lddl] receives (softmax - onehot)/M (columns V..lddl-1 zeroed),
 * i.e. the gradient of the loss w.r.t. the logits.  labels: int64 [M] in [0, V). */
PGNN_API int pgnn_softmax_ce_fwd(const float* logits, int64_t ld, int64_t M, int64_t V, const int64_t* labels,
                                 double* loss_mean, float* dlogits, int64_t lddl, void* stream);
/* The same loss with each label given as a row of Q floats (label_rows [M, ld_label]): the label of row m is the FIRST index
 * of the maximum of its Q values, `torch.argmax(batch.mask_edge_label, dim=1)` followed by CrossEntropyLoss of bio masking
 * (bio/pretrain_masking.py:47-55: V = 7 edge types, Q = 9 attribute columns; evaluated in fp64).  A label >= V, or a row
 * without a finite maximum (a NaN in it, or a +-Inf maximum), sets PGNN_DEVERR_LABEL and the row contributes its
 * log-sum-exp only, as an out-of-range int64 label does above.  *loss_mean is OVERWRITTEN, dlogits as above.  Deterministic
 * (per-CTA fp64 partials folded in order, no floating-point atomics).  workspace: pgnn_softmax_ce_rows_workspace_bytes()
 * bytes, any content. */
PGNN_API int64_t pgnn_softmax_ce_rows_workspace_bytes(void);
PGNN_API int pgnn_softmax_ce_rows_fwd(const float* logits, int64_t ld, int64_t M, int64_t V, const float* label_rows, int64_t ld_label,
                                      int64_t Q, double* loss_mean, float* dlogits, int64_t lddl, void* workspace,
                                      int64_t workspace_bytes, void* stream);
/* Edge-prediction head (chem/pretrain_edgepred.py:31-41, bio/pretrain_edgepred.py): over x [N, ldx] fp32 (C columns),
 *   pos_scores[p] = <x[pos_u[p * pos_stride]], x[pos_v[p * pos_stride]]>  (p < P; pos_u / pos_v: the two rows of
 *                   edge_index[:, ::2], column stride pos_stride, no copy), neg_scores[q] likewise over the Q negative pairs,
 *   *loss = mean_p BCE(pos_p, 1) + mean_q BCE(neg_q, 0)  (fp64; an empty side contributes NaN, as torch's empty mean does).
 * Each dot product is an fp32 fmaf chain in a fixed order; dscore [P + Q] receives d loss / d score ((sigmoid - t) / P, then
 * / Q); pairs [2, P + Q] int64 receives the pairs (positives first) for pgnn_graph_prep.  A pair with an endpoint outside
 * [0, N) scores 0 and sets PGNN_DEVERR_GATHER.  C and ldx must be multiples of 4 and x 16-byte aligned.  Deterministic (per-CTA
 * fp64 partials folded in order).  workspace: pgnn_edge_pair_bce_workspace_bytes() bytes, any content. */
PGNN_API int64_t pgnn_edge_pair_bce_workspace_bytes(void);
PGNN_API int pgnn_edge_pair_bce_fwd(const float* x, int64_t ldx, int64_t N, int64_t C, const int64_t* pos_u, const int64_t* pos_v,
                                    int64_t pos_stride, int64_t P, const int64_t* neg_u, const int64_t* neg_v, int64_t neg_stride,
                                    int64_t Q, double* loss, float* pos_scores, float* neg_scores, float* dscore, int64_t* pairs,
                                    void* workspace, int64_t workspace_bytes, void* stream);
/* Its backward: gx[i] = sum_{p: u_p = i} g_p x[v_p] + sum_{p: v_p = i} g_p x[u_p] with g_p = dscore[p] * (float)*gscale (gscale:
 * device fp64 scalar, the gradient of the loss), each sum in pair order.  rowptr/nbr/eid _t and _s: pgnn_graph_prep of the
 * `pairs` list over N nodes.  gx [N, ldgx] is OVERWRITTEN.  Deterministic, no atomics. */
PGNN_API int pgnn_edge_pair_bce_bwd(const float* x, int64_t ldx, int64_t N, int64_t C, const float* dscore, const double* gscale,
                                    const int32_t* rowptr_t, const int32_t* nbr_t, const int32_t* eid_t, const int32_t* rowptr_s,
                                    const int32_t* nbr_s, const int32_t* eid_s, float* gx, int64_t ldgx, void* stream);
/* Deep Graph Infomax head (chem/pretrain_deepgraphinfomax.py:61-73, bio/pretrain_deepgraphinfomax.py), csrc/infomax.cu.  Over
 * node rows x [N, ldx] fp32 (C columns) of G graphs (batch: int64 [N] graph ids; seg_ptr [G+1] / seg_order [N] from
 * pgnn_bucket(batch), as for pgnn_segment_mean_fwd; an id outside [0, G) has pgnn_bucket's precondition) and the
 * Discriminator weight W [C, C] (contiguous):
 *   S = sigmoid(segment mean of x)             [G, C]   pgnn_infomax_summary_fwd (an empty graph gives sigmoid(0) = 0.5)
 *   H = S . W                                  [G, C]   the caller: pgnn_linear_bwd_x(gy = S, w = W)
 *   pos[i] = <x_i, H[b_i]>, neg[i] = <x_i, H[(b_i + 1) mod G]>   (cycle_index(G, 1); G = 1 pairs a graph with itself)
 *   *loss = mean_i BCE(pos_i, 1) + mean_i BCE(neg_i, 0)          pgnn_infomax_bce_fwd (fp64; N = 0 gives NaN)
 * Each score is an fp32 fmaf chain over float4 columns in a fixed order; dscore [2N] receives d loss / d score ((sigmoid - 1) / N
 * for pos, then sigmoid / N for neg).  H [G, C] contiguous.  C and ldx must be multiples of 4 and x, H 16-byte aligned (else
 * PGNN_EUNSUPPORTED).  Deterministic (per-CTA fp64 partials folded in order).  workspace: pgnn_infomax_bce_workspace_bytes()
 * bytes, any content. */
PGNN_API int pgnn_infomax_summary_fwd(const float* x, int64_t ldx, const int32_t* seg_ptr, const int32_t* seg_order, int64_t G,
                                      int64_t C, float* S, int64_t lds, void* stream);
PGNN_API int64_t pgnn_infomax_bce_workspace_bytes(void);
PGNN_API int pgnn_infomax_bce_fwd(const float* x, int64_t ldx, int64_t N, int64_t C, const int64_t* batch, const float* H, int64_t G,
                                  double* loss, float* pos, float* neg, float* dscore, void* workspace, int64_t workspace_bytes,
                                  void* stream);
/* Its backward, with gscale the device fp64 upstream gradient of the loss (S, H as the forward left them, contiguous [G, C]):
 *   dH[g] = gscale (sum_{i in g} dpos_i x_i + sum_{i in prev(g)} dneg_i x_i), prev(g) = (g - 1) mod G, rows in seg_order's
 *           stable order, 8 partials per graph folded in order (no atomics);
 *   gW    = S^T . dH   (pgnn_linear_bwd_w(gy = S, x = dH); at precision 1 its 3xTF32 GEMM with the split-K partials in the
 *           workspace, folded in order);  dS = dH . W^T   (pgnn_linear_fwd(x = dH, w = W));
 *   gx_i  = gscale (dpos_i H[b_i] + dneg_i H[(b_i + 1) mod G]) + dS[b_i] * S[b_i] * (1 - S[b_i]) / n_{b_i}, one pass.
 * gx [N, ldgx] and gW [C, C] are OVERWRITTEN; either may be NULL (not computed).  precision as for pgnn_linear_*.  At 1 every
 * output repeats bit for bit; at 0 gW inherits the FFMA weight-gradient GEMM's split-K atomics (G > 64: rounding-level jitter).
 * workspace: pgnn_infomax_bce_bwd_workspace_bytes(G, C) bytes, 16-byte aligned, any content. */
PGNN_API int64_t pgnn_infomax_bce_bwd_workspace_bytes(int64_t G, int64_t C);
PGNN_API int pgnn_infomax_bce_bwd(const float* x, int64_t ldx, int64_t N, int64_t C, const int64_t* batch, const int32_t* seg_ptr,
                                  const int32_t* seg_order, int64_t G, const float* S, const float* H, const float* W,
                                  const float* dscore, const double* gscale, float* gx, int64_t ldgx, float* gW, int precision,
                                  void* workspace, int64_t workspace_bytes, void* stream);
/* out[r] = sum_d a[r,d] * b[(r + shift) mod B, d]   (cycle_index negatives, pretrain_contextpred.py:36-39,64-67) */
PGNN_API int pgnn_shifted_rowdot_fwd(const float* a, int64_t lda, const float* b, int64_t ldb, int64_t B, int64_t C,
                                     int64_t shift, float* out, void* stream);
/* ga[r,:] (+)= g[r] * b[(r+shift)%B,:] ; gb[r,:] (+)= g[(r-shift)%B] * a[(r-shift)%B,:] ; accumulate != 0 adds */
PGNN_API int pgnn_shifted_rowdot_bwd(const float* g, const float* a, int64_t lda, const float* b, int64_t ldb,
                                     int64_t B, int64_t C, int64_t shift, int accumulate,
                                     float* ga, int64_t ldga, float* gb, int64_t ldgb, void* stream);
/* Mean binary cross-entropy with logits over fp32 logits [M,N] evaluated in fp64 (BCEWithLogitsLoss on pred.double()):
 *   target_kind 0: every target = const_target         (chem/pretrain_contextpred.py:86-87: ones for pred_pos, zeros for pred_neg)
 *   target_kind 1: target int64 [M, ldt] in {0,1}      (bio/pretrain_supervised.py:33-36: go_target_pretrain)
 *   target_kind 2: target int64 in {-1,0,+1}; 0 = missing label, dropped; the rest use (y+1)/2; loss = sum / #valid
 *                                                      (chem/finetune.py:33-43)
 * *loss_mean (device fp64 scalar) is OVERWRITTEN; dlogits [M, lddl] receives d loss / d logits (0 at dropped entries).
 * Deterministic (no floating-point atomics).  workspace: pgnn_bce_logits_workspace_bytes() bytes, any content. */
PGNN_API int64_t pgnn_bce_logits_workspace_bytes(void);
PGNN_API int pgnn_bce_logits_fwd(const float* logits, int64_t ld, int64_t M, int64_t N, const int64_t* target, int64_t ldt,
                                 int target_kind, double const_target, double* loss_mean, float* dlogits, int64_t lddl,
                                 void* workspace, int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Whole-encoder entry points: chem GNN with gnn_type="gin", JK="last" (chem/model.py:255-290).  pgnn_chem_gin_* run without
 * dropout; pgnn_chem_encoder_forward / _backward below are the same path for every gnn_type with live dropout.
 * What GNN.forward / loss.backward() bind to: two boundary crossings per training step.
 *
 * params: HOST array of num_params = 2 + 8*L DEVICE pointers in state_dict order
 *   [x_embedding1.weight, x_embedding2.weight,
 *    then per layer l: gnns.l.mlp.0.weight, .mlp.0.bias, .mlp.2.weight, .mlp.2.bias,
 *                      gnns.l.edge_embedding1.weight, .edge_embedding2.weight, batch_norms.l.weight, .bias]
 * bn_running_mean / bn_running_var / bn_num_batches_tracked: HOST arrays of L device pointers (updated in
 *   training mode exactly as torch.nn.BatchNorm1d does; bn_num_batches_tracked may be NULL).
 * workspace: device scratch of pgnn_chem_gin_workspace_bytes; forward leaves the bucketed graph and the saved
 *   activations in it, backward consumes them, so the SAME workspace must be passed to both.
 * precision: backward must get the forward's (what the forward saves depends on it: the tensor-path backward reads the one-hot
 *   atom-code rows that only a precision = 1 training forward writes).
 * grads: ONE flat fp32 buffer; tensor i of the params order lives at [offsets[i], offsets[i+1]) with offsets from
 *   pgnn_chem_gin_grad_offsets (host array of num_params + 1 entries).  OVERWRITTEN.
 * ------------------------------------------------------------------------------------------- */
PGNN_API int64_t pgnn_chem_gin_num_params(int64_t L);
PGNN_API int pgnn_chem_gin_grad_offsets(int64_t L, int64_t D, int64_t* offsets);
PGNN_API int64_t pgnn_chem_gin_workspace_bytes(int64_t N, int64_t E, int64_t L, int64_t D);
/* test aid: byte offsets in the workspace of z1 [L][N][2D] (post-ReLU hidden), z2 [L][N][D] (pre-BatchNorm), BatchNorm batch mean
 * [L][D] and invstd [L][D] after a training forward: lets a test recover the ReLU decisions the encoder took */
PGNN_API int pgnn_chem_gin_debug_layout(int64_t N, int64_t E, int64_t L, int64_t D, int64_t* out4);
/* test aid: byte offset in the same workspace of aggr [L][N][D], layer l's gathered input after a training forward (for l > 0 the
 * previous layer's BatchNorm + ReLU as the gather applied it on load); PGNN_EINVAL for bad sizes */
PGNN_API int64_t pgnn_chem_gin_debug_aggr_offset(int64_t N, int64_t E, int64_t L, int64_t D);
/* test aids for the 3xTF32 wgmma GEMM (precision 1), reachable here with every operand layout, tile width and epilogue:
 *   pgnn_debug_tc_gemm: C[m,n] = sum_r A(m,r) B(n,r), r < K.  a_kc / b_kc != 0: the operand is reduction-contiguous
 *     (A(m,r) = A[m*lda + r]), else A(m,r) = A[r*lda + m] (same for B with n).  bn = the tile width, 64 or 128.  Epilogue as in
 *     the encoders: + bias[N], relu != 0 (NaN kept), mask [M, ldm] (0 where mask <= 0 or NaN); then, all accumulated with
 *     atomics into caller-zeroed buffers, colsum[N] += column sums, stats[2][N] += fp64 sums and sums of squares,
 *     gT[q][n] (q < q_split) / gT2[q - q_split][n] (q >= q_split), row stride ldt, += sum_m S[m*Q + q] C[m,n] for 1 <= Q <= 16.
 *     Optional pointers may be NULL.  PGNN_EUNSUPPORTED when lda or ldb is not a multiple of 4 or A / B is not 16-byte aligned.
 *   pgnn_debug_tc_wgrad: gw[N,K] = gy[M,N]^T . x[M,K], gb[N] = column sums of gy (may be NULL), split-K over the M rows: with
 *     partials (16-byte aligned, >= splits*N*K floats, N*K % 4 == 0) each split stores a partial tile and one kernel folds them
 *     in split order; otherwise the splits accumulate with atomics.
 *   pgnn_debug_tc_wgrad_plan: host only; out4 = {tile width, output tiles, splits, rows per split} of that GEMM.
 *   pgnn_debug_transpose_batch: out[i] [cols[i], rows[i]] = transpose of in[i] [rows[i], cols[i]] for count <= 32 jobs (HOST arrays
 *     of device pointers and sizes); PGNN_EUNSUPPORTED above 32. */
PGNN_API int pgnn_debug_tc_gemm(int a_kc, int b_kc, int bn, const float* A, int64_t lda, const float* B, int64_t ldb, float* C,
                                int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias, int relu, const float* mask,
                                int64_t ldm, float* colsum, double* stats, const float* S, int Q, float* gT, float* gT2,
                                int q_split, int64_t ldt, void* stream);
PGNN_API int pgnn_debug_tc_wgrad(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t N, int64_t K,
                                 float* gw, float* gb, float* partials, int64_t partial_floats, void* stream);
PGNN_API int pgnn_debug_tc_wgrad_plan(int64_t M, int64_t N, int64_t K, int64_t* out4);
PGNN_API int pgnn_debug_transpose_batch(int count, const float* const* in, float* const* out, const int32_t* rows,
                                        const int32_t* cols, void* stream);
/* test aids for the weight-image path of the same GEMM (the forward and dgrad GEMMs of the chem GIN encoder): a weight used as a
 * reduction-contiguous B [rows, K] is split into tf32 hi / lo once and stored as two planes, hi then lo, each
 * [ceil(rows / 128) * 128][ceil(K / 32) * 32] floats row-major (image floats = 2 x that); inside every 32-wide block of a row, slot
 * s holds element k = kperm(s) = (s & 16) | ((s & 3) << 2) | ((s >> 2) & 3) of the block; padding is zero.  hi = x + 0 with its low
 * 13 bits cleared, lo = x - hi (fp32).
 *   pgnn_debug_pack_weight_images: count <= 32 images in one launch (HOST arrays): job i reads w[i] [rows[i], cols[i]] with row
 *     stride ld[i] >= cols[i] and writes into img[i] (16-byte aligned) the image of w[i] (transposed[i] == 0: B rows = rows[i],
 *     K = cols[i]) or of its transpose (B rows = cols[i], K = rows[i]).  PGNN_EUNSUPPORTED above 32 jobs.
 *   pgnn_debug_tc_gemm_img: pgnn_debug_tc_gemm with a_kc = b_kc = 1 (same arguments and epilogue, bit for bit the same result)
 *     through the image path: packs B [N, K] into img (16-byte aligned, image floats of N rows and K) and runs the GEMM from it. */
PGNN_API int pgnn_debug_pack_weight_images(int count, const float* const* w, const int64_t* ld, const int32_t* rows,
                                           const int32_t* cols, const int32_t* transposed, float* const* img, void* stream);
PGNN_API int pgnn_debug_tc_gemm_img(int bn, const float* A, int64_t lda, const float* B, int64_t ldb, float* img, float* C,
                                    int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias, int relu, const float* mask,
                                    int64_t ldm, float* colsum, double* stats, const float* S, int Q, float* gT, float* gT2,
                                    int q_split, int64_t ldt, void* stream);
/* test aids for the two BatchNorm sweeps only the whole encoder reaches (dropout of (drop_p, drop_seed, drop_layer) as in
 * pgnn_dropout_fwd; drop_p = 0 runs the mask-free kernels):
 *   pgnn_debug_bn_apply_fold: pgnn_bn_fwd_train's finalisation and apply in one kernel, from raw fp64 sums[2][C] (sum, sum of
 *     squares of the M rows of x).  Every CTA derives scale / shift itself (invstd = 1 / sqrtf((float)var + eps)); CTA 0 alone
 *     writes save_mean / save_invstd and updates running_mean / running_var / *num_batches_tracked (each may be NULL).
 *     C <= 6144 (scale / shift live in 48 KiB of shared memory).
 *   pgnn_debug_bn_bwd_colsum: pgnn_bn_bwd (mask applied to gy before the ReLU mask) that also leaves the column sums of gx in
 *     colsum[C] (OVERWRITTEN).  Row strides ldgy, ldx, ldgx >= C. */
PGNN_API int pgnn_debug_bn_apply_fold(const float* x, int64_t ldx, int64_t M, int64_t C, const double* sums, const float* gamma,
                                      const float* beta, float* running_mean, float* running_var, int64_t* num_batches_tracked,
                                      float momentum, float eps, float* save_mean, float* save_invstd, int relu, float* y, int64_t ldy,
                                      float drop_p, int64_t drop_seed, int64_t drop_layer, void* stream);
PGNN_API int pgnn_debug_bn_bwd_colsum(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t C,
                                      const float* gamma, const float* beta, const float* save_mean, const float* save_invstd, int relu,
                                      float* gx, int64_t ldgx, float* ggamma, float* gbeta, float* colsum, float drop_p,
                                      int64_t drop_seed, int64_t drop_layer, void* workspace, int64_t workspace_bytes, void* stream);
PGNN_API int pgnn_chem_gin_forward(const void* const* params, void* const* bn_running_mean, void* const* bn_running_var,
                                   void* const* bn_num_batches_tracked, const int64_t* x, const int64_t* edge_index,
                                   const int64_t* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D, int training,
                                   float momentum, float eps, int precision, float* node_rep, int64_t ld_out,
                                   void* workspace, int64_t workspace_bytes, void* stream);
PGNN_API int pgnn_chem_gin_backward(const void* const* params, const float* g_node_rep, int64_t ldg, const int64_t* x,
                                    int64_t N, int64_t E, int64_t L, int64_t D, int precision, float* grads,
                                    void* workspace, int64_t workspace_bytes, void* stream);

/* The same two-call contract for gnn_type = "gcn" | "graphsage" | "gat" (chem/model.py:58-202 inside GNN.forward :255-290).
 * params order: [x_embedding1.weight, x_embedding2.weight, then per layer
 *   gcn / graphsage: gnns.l.linear.weight [D,D], .linear.bias, .edge_embedding1.weight [6,D], .edge_embedding2.weight [3,D],
 *                    batch_norms.l.weight, .bias                                                         (6 per layer)
 *   gat (heads = 2): gnns.l.weight_linear.weight [2D,D], .weight_linear.bias [2D], .att [1,2,2D], .bias [D],
 *                    .edge_embedding1.weight [6,2D], .edge_embedding2.weight [3,2D], batch_norms.l.weight, .bias  (8 per layer)]
 * The flat gradient buffer uses the same order (pgnn_chem_conv_grad_offsets).  backward also takes edge_attr (GAT re-reads the
 * bond codes); everything else as for pgnn_chem_gin_*. */
#define PGNN_CONV_GCN 1
#define PGNN_CONV_SAGE 2
#define PGNN_CONV_GAT 3
PGNN_API int64_t pgnn_chem_conv_num_params(int conv_type, int64_t L);
PGNN_API int pgnn_chem_conv_grad_offsets(int conv_type, int64_t L, int64_t D, int64_t* offsets);
PGNN_API int64_t pgnn_chem_conv_workspace_bytes(int conv_type, int64_t N, int64_t E, int64_t L, int64_t D);
PGNN_API int pgnn_chem_conv_forward(int conv_type, const void* const* params, void* const* bn_running_mean,
                                    void* const* bn_running_var, void* const* bn_num_batches_tracked, const int64_t* x,
                                    const int64_t* edge_index, const int64_t* edge_attr, int64_t N, int64_t E, int64_t L,
                                    int64_t D, int training, float momentum, float eps, int precision, float* node_rep,
                                    int64_t ld_out, void* workspace, int64_t workspace_bytes, void* stream);
PGNN_API int pgnn_chem_conv_backward(int conv_type, const void* const* params, const float* g_node_rep, int64_t ldg,
                                     const int64_t* x, const int64_t* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D,
                                     int precision, float* grads, void* workspace, int64_t workspace_bytes, void* stream);

/* The one implementation behind pgnn_chem_gin_* (gnn_type 0) and pgnn_chem_conv_* (gnn_type = PGNN_CONV_*), with the reference's
 * dropout (chem/model.py:271-275): in training mode with drop_p > 0, layer l's output (after its BatchNorm and, except for the
 * last layer, its ReLU) is multiplied by the pgnn_dropout_fwd mask of (drop_p, drop_seed, layer = l).  It never makes a pass of
 * its own: the kernel that writes or loads layer l's output applies it (GIN: the next layer's gather and the BatchNorm apply of
 * node_rep; the conv types: the BatchNorm apply that writes the layer's output), and the backward applies it to the incoming
 * gradient inside the BatchNorm backward.  Eval mode (training = 0) applies none; backward must get the forward's drop_p,
 * drop_seed and precision.  drop_p == 0 is exactly pgnn_chem_gin_* / pgnn_chem_conv_*, which pass it.  Workspace, parameter and gradient
 * layouts are those of the type's own entry points; backward's edge_attr is only read for GAT.  gnn_type outside {0, 1, 2, 3},
 * drop_p outside [0, 1] or NaN: PGNN_EINVAL. */
PGNN_API int pgnn_chem_encoder_forward(int gnn_type, const void* const* params, void* const* bn_running_mean,
                                       void* const* bn_running_var, void* const* bn_num_batches_tracked, const int64_t* x,
                                       const int64_t* edge_index, const int64_t* edge_attr, int64_t N, int64_t E, int64_t L,
                                       int64_t D, int training, float momentum, float eps, float drop_p, int64_t drop_seed,
                                       int precision, float* node_rep, int64_t ld_out, void* workspace, int64_t workspace_bytes,
                                       void* stream);
PGNN_API int pgnn_chem_encoder_backward(int gnn_type, const void* const* params, const float* g_node_rep, int64_t ldg,
                                        const int64_t* x, const int64_t* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D,
                                        float drop_p, int64_t drop_seed, int precision, float* grads, void* workspace,
                                        int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Whole-encoder entry points of the bio GNN (bio/model.py:11-290, JK="last", any drop_ratio): the same two-call contract as
 * pgnn_chem_encoder_* for gnn_type 0 = GIN and PGNN_CONV_GCN / _SAGE / _GAT.
 *
 * Per layer: layer 0 embeds the dummy label x [N] (float-coded 0 / 1) with input_node_embeddings [2, D].  Each conv's edge encoder
 * Linear(9, C) (C = 2D for GAT, else D) acts through the summary S [N,10] of pgnn_bio_edge_summary (self-loop bit at column 7); the
 * library builds its [10, C] table [W^T ; b] itself.
 *   GIN:  message [x_j || e_ij] (2D wide), MLP Linear(2D,2D) -> BatchNorm1d(2D) -> ReLU -> Linear(2D,D);
 *   GCN / GraphSAGE (+ L2 normalisation) / GAT (2 heads, slope 0.2): Linear, then the conv as in the chem block.
 * There is no outer BatchNorm.  Every layer but the last is followed by ReLU; in training with drop_p > 0, layer l's output is then
 * multiplied by the pgnn_dropout_fwd mask of (drop_p, drop_seed, layer = l).  Eval mode (training = 0) applies none.
 *
 * params: HOST array of num_params = 1 + P*L DEVICE pointers
 *   [gnns.0.input_node_embeddings.weight [2,D], then per layer gnns.l.
 *    gin  (P = 8): mlp.0.weight [2D,2D], mlp.0.bias [2D], mlp.1.weight [2D], mlp.1.bias [2D], mlp.3.weight [D,2D], mlp.3.bias [D],
 *                  edge_encoder.weight [D,9], edge_encoder.bias [D]
 *    gcn / graphsage (P = 4): linear.weight [D,D], linear.bias [D], edge_encoder.weight [D,9], edge_encoder.bias [D]
 *    gat  (P = 6): weight_linear.weight [2D,D], weight_linear.bias [2D], att [1,2,2D], bias [D], edge_encoder.weight [2D,9],
 *                  edge_encoder.bias [2D]]
 * bn_running_mean / bn_running_var / bn_num_batches_tracked: HOST arrays of L device pointers, the inner BatchNorm1d(2D) of each
 *   GIN layer (gnns.l.mlp.1), updated in training mode as torch does; num_batches_tracked may be NULL.  Ignored (may be NULL) for
 *   the other types.
 * workspace: pgnn_bio_encoder_workspace_bytes; the SAME workspace goes to forward and backward.  The backward must get the
 *   forward's drop_p, drop_seed and precision.
 * grads: ONE flat fp32 buffer, tensor i of the params order (in the parameter's own shape) at [offsets[i], offsets[i+1]) of
 *   pgnn_bio_encoder_grad_offsets (host array of num_params + 1 entries).  OVERWRITTEN.  backward's edge_attr is only read for GAT.
 * D % 4 == 0.  gnn_type outside {0, 1, 2, 3}, L < 1, drop_p outside [0, 1] or NaN: PGNN_EINVAL.  A short workspace: PGNN_EWORKSPACE.
 * ------------------------------------------------------------------------------------------- */
PGNN_API int64_t pgnn_bio_encoder_num_params(int gnn_type, int64_t L);
PGNN_API int pgnn_bio_encoder_grad_offsets(int gnn_type, int64_t L, int64_t D, int64_t* offsets);
PGNN_API int64_t pgnn_bio_encoder_workspace_bytes(int gnn_type, int64_t N, int64_t E, int64_t L, int64_t D);
PGNN_API int pgnn_bio_encoder_forward(int gnn_type, const void* const* params, void* const* bn_running_mean,
                                      void* const* bn_running_var, void* const* bn_num_batches_tracked, const float* x /*[N]*/,
                                      const int64_t* edge_index, const float* edge_attr /*[E,9]*/, int64_t N, int64_t E, int64_t L,
                                      int64_t D, int training, float momentum, float eps, float drop_p, int64_t drop_seed,
                                      int precision, float* node_rep, int64_t ld_out, void* workspace, int64_t workspace_bytes,
                                      void* stream);
PGNN_API int pgnn_bio_encoder_backward(int gnn_type, const void* const* params, const float* g_node_rep, int64_t ldg,
                                       const float* x, const float* edge_attr, int64_t N, int64_t E, int64_t L, int64_t D,
                                       float drop_p, int64_t drop_seed, int precision, float* grads, void* workspace,
                                       int64_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Either side of the path inside a training step (SURVEY.md section 8(f): f1 collation, f2 optimizer).
 * ------------------------------------------------------------------------------------------- */
/* Device-side batch collation for chem graphs: what BatchMasking.from_data_list / BatchSubstructContext do on the host
 * (chem/batch.py:17-52: concatenate per-graph tensors, add the running node count to edge_index, build `batch`).
 * The molecule store is resident in HBM in compact form:
 *   node_ptr[G+1], edge_ptr[G+1]  int64 prefix sums of atoms / directed bonds per graph
 *   store_x[2*Nt] uint8 (atom type, chirality), store_edge_attr[2*Et] uint8 (bond type, direction), both row-major [.,2]
 *   store_edge_index[2][Et] int32, graph-LOCAL endpoints (row 0 then row 1, as edge_index)
 * graph_ids[B] int64 selects and orders the graphs of the batch.  Outputs (sizes N = sum n_g, E = sum e_g, which the host
 * knows from its copy of the prefix sums): x [N,2], edge_index [2,E], edge_attr [E,2], batch [N], all int64 as GNN.forward
 * takes them; node_off / edge_off [B+1] int64 receive the exclusive scans (node_off is the per-graph offset the reference
 * adds to masked_atom_indices, chem/batch.py:40-45).  Bit-exact. */
PGNN_API int pgnn_collate_chem(const int64_t* node_ptr, const int64_t* edge_ptr, const uint8_t* store_x,
                               const int32_t* store_edge_index, int64_t store_num_edges, const uint8_t* store_edge_attr,
                               const int64_t* graph_ids, int64_t B, int64_t* node_off, int64_t* edge_off, int64_t* x,
                               int64_t* edge_index, int64_t* edge_attr, int64_t* batch, void* stream);

/* MaskAtom (chem/util.py:189-241, mask_edge=False) on a collated batch: per graph int(n * mask_rate + 1) distinct atoms (uniform
 * k-subset: the k smallest splitmix64(seed, position-in-batch) keys of the graph), labels saved, x rows overwritten with
 * [mask_token, 0] (mask_token = num_atom_type = 119, chem/pretrain_masking.py:122).  x [N,2] int64 is modified IN PLACE;
 * node_off [B+1] as written by pgnn_collate_chem.  Outputs: mask_off [B+1] (exclusive scan of the sample sizes),
 * masked_atom_indices [M] (batch-global node ids, ascending inside a graph), mask_node_label [M,2]; M =
 * pgnn_mask_atoms_count(host copy of node_off, B, mask_rate).  Integer work, bit-exact against oracle/step_io_oracle.py.
 * mask_edge=True: follow with pgnn_mask_edges_chem. */
PGNN_API int64_t pgnn_mask_atoms_count(const int64_t* node_off_host, int64_t B, double mask_rate);
PGNN_API int pgnn_mask_atoms(int64_t* x, const int64_t* node_off, int64_t B, double mask_rate, int64_t mask_token, int64_t seed,
                             int64_t* mask_off, int64_t* masked_atom_indices, int64_t* mask_node_label, void* stream);
/* Per-graph index lists of a batch (chem/batch.py:41-42,170-199; bio/batch.py:39-40): the store holds list_ptr [G+1] int64 and
 * values int32 (graph-local node ids); for the selected graphs out[list_off[i] + j] = values[list_ptr[g_i] + j] +
 * add_per_graph[i] (e.g. node_off of the same collation; NULL = 0), seg[...] = i (batch_overlapped_context; may be NULL),
 * sizes[i] = list length (overlapped_context_size; may be NULL).  list_off [B+1] receives the exclusive scan. */
PGNN_API int pgnn_collate_lists(const int64_t* list_ptr, const int32_t* values, const int64_t* graph_ids, int64_t B,
                                const int64_t* add_per_graph, int64_t* list_off, int64_t* out, int64_t* seg, int64_t* sizes,
                                void* stream);
/* bio/batch.py:17-50 for a store of PPI ego graphs: node_ptr / edge_ptr [G+1], store_edge_index [2][Et] int32 graph-local,
 * store_edge_bits [Et] uint16 = the 9 binary edge attributes of bio/loader.py:57-75 packed LSB-first.  Outputs: x float [N,1]
 * (the constant dummy label 1.0, bio/loader.py:47), edge_index int64 [2,E] with the node offset added, edge_attr float [E,9],
 * batch int64 [N], node_off / edge_off [B+1]. */
PGNN_API int pgnn_collate_bio(const int64_t* node_ptr, const int64_t* edge_ptr, const int32_t* store_edge_index,
                              int64_t store_num_edges, const uint16_t* store_edge_bits, const int64_t* graph_ids, int64_t B,
                              int64_t* node_off, int64_t* edge_off, float* x, int64_t* edge_index, float* edge_attr,
                              int64_t* batch, void* stream);

/* The mask_edge=True half of MaskAtom (chem/util.py:243-272) on a collated batch whose atoms pgnn_mask_atoms has masked:
 * per graph L = the edge columns with an endpoint in masked_atom_indices [M] (batch-global node ids), ascending;
 * connected_edge_indices = L[::2] (+ the edge offset, chem/batch.py:41-42), mask_edge_label = edge_attr[L[::2]] (read before
 * the overwrite), edge_attr[L] = [num_edge_type, 0] in place.  edge_index [2,E], edge_attr [E,2] int64; edge_off [B+1] as written
 * by pgnn_collate_chem; conn_off [B+1] receives the exclusive scan of the per-graph list lengths (conn_off[B] = the total the
 * host reads back); the two outputs must hold E/2 + B entries (rows).  Bit-exact against oracle/step_io_oracle.mask_edges_chem. */
PGNN_API int64_t pgnn_mask_edges_chem_workspace_bytes(int64_t N, int64_t B);
PGNN_API int pgnn_mask_edges_chem(const int64_t* edge_index, int64_t* edge_attr, const int64_t* edge_off, int64_t B, int64_t N,
                                  int64_t E, const int64_t* masked_atom_indices, int64_t M, int64_t num_edge_type,
                                  void* workspace, int64_t workspace_bytes, int64_t* conn_off, int64_t* connected_edge_indices,
                                  int64_t* mask_edge_label, void* stream);
/* MaskEdge (bio/util.py:46-104) on a batch collated by pgnn_collate_bio: per graph int(e/2 * mask_rate + 1) distinct bond pairs
 * (uniform k-subset: the k smallest splitmix64(seed, column id) keys), masked_edge_idx [M] = their first columns (ascending, edge
 * offset included: bio/batch.py:95-96), mask_edge_label [M,9] = their attribute rows, then both directions of each pair set to
 * [0,0,0,0,0,0,0,0,1] in place.  M = pgnn_mask_edges_bio_count(host copy of edge_off, B, mask_rate); mask_off [B+1] receives
 * the exclusive scan of the sample sizes.  Bit-exact against oracle/step_io_oracle.mask_edges_bio. */
PGNN_API int64_t pgnn_mask_edges_bio_count(const int64_t* edge_off_host, int64_t B, double mask_rate);
PGNN_API int pgnn_mask_edges_bio(float* edge_attr, const int64_t* edge_off, int64_t B, double mask_rate, int64_t seed,
                                 int64_t* mask_off, int64_t* masked_edge_idx, float* mask_edge_label, void* stream);
/* NegativeEdge (chem/util.py:22-52, bio/util.py:16-44) + BatchAE's node offset (chem/batch.py:69-121) on a batch collated by
 * pgnn_collate_chem / pgnn_collate_bio (edge_index [2,E] int64 batch-global, node_off / edge_off [B+1]).  Per graph of n nodes
 * and e columns, candidate j < 5e is (splitmix64(seed, 2 (5 edge_off[g] + j)) mod n, splitmix64(seed, 2 (5 edge_off[g] + j) + 1)
 * mod n); it is accepted iff its endpoints differ, it is not a (directed) column of the graph and was not accepted before; the
 * walk stops once e/2 are accepted when e is even (never when e is odd; n = 0 or e = 0 draws nothing).  negative_edge_index
 * receives the accepted pairs + the graph's node offset as a contiguous [2, M] at its front (it must hold 2 * capacity int64),
 * negative_edge_off [B+1] the exclusive scan of the per-graph counts (negative_edge_off[B] = M, the value the host reads back).
 * capacity = pgnn_negative_edges_capacity(host copy of edge_off, B) = sum_g (e_g even ? e_g / 2 : 5 e_g).  A column endpoint
 * outside its graph is ignored and sets PGNN_DEVERR_GATHER.  The workspace is linear in B, E and capacity.  Bit-exact against
 * the host restatement of tests/edgepred_oracle.py. */
PGNN_API int64_t pgnn_negative_edges_capacity(const int64_t* edge_off_host, int64_t B);
PGNN_API int64_t pgnn_negative_edges_workspace_bytes(int64_t B, int64_t E, int64_t capacity);
PGNN_API int pgnn_negative_edges(const int64_t* edge_index, int64_t E, const int64_t* node_off, const int64_t* edge_off, int64_t B,
                                 int64_t seed, int64_t capacity, void* workspace, int64_t workspace_bytes, int64_t* negative_edge_index,
                                 int64_t* negative_edge_off, void* stream);

/* ExtractSubstructureContextPair + BatchSubstructContext.from_data_list on the device (chem/util.py:55-151 through
 * chem/loader.py:146-221, chem/batch.py:141-210; bio/util.py:123-205, bio/batch.py:196-265) for graphs held in HBM.
 * Per selected graph i (root r_i = roots[i], graph-local; roots == NULL: r_i = splitmix64(seed, i) mod n_i, a uniform draw --
 * the reference's random.sample cannot be matched bit for bit): d(v) = hop distance from r_i in the undirected graph of the
 * even-indexed edge columns (pair p = columns 2p, 2p+1; pair_first[p] = 0 marks a pair whose endpoints already occurred and
 * which networkx therefore ignores, chem/loader.py:173; every graph must hold an even number of columns);
 *   whole_graph = 0 (chem): substructure = {d <= k}, context = {d <= l1} xor {d <= l2}, a cutoff <= 0 meaning {root};
 *   whole_graph = 1 (bio):  substructure = the whole graph, context = {d > l1} (k, l2 ignored);
 * overlap = substructure & context; a graph with an empty context is dropped from the batch (chem/batch.py:168).
 * pgnn_extract_pairs runs the BFS and the scans: offsets [6][B+1] int64 receives the exclusive scans over the batch of
 * (substructure nodes, substructure edge columns, context nodes, context edge columns, overlap entries, kept flag);
 * offsets[q][B] are the totals the host reads back to size its views.  pgnn_extract_fill_{chem,bio} then write the batch:
 * nodes renumbered ascending by original index, both directions of a kept pair adjacent ((i,j),(j,i), the attribute row of
 * column 2p), edge_index compact [2, total], centre / overlap indices offset by their side's running node count,
 * batch_overlapped_context = ordinal among the kept graphs.  Output buffers must hold the upper bounds: full_nodes rows and
 * the selected graphs' full edge-column count.  full_nodes = sum of n_i (the host knows it from its copy of node_ptr).
 * Integer work, bit-exact against oracle/step_io_oracle.extract_pairs_batch. */
PGNN_API int64_t pgnn_extract_pairs_workspace_bytes(int64_t B, int64_t full_nodes);
PGNN_API int pgnn_extract_pairs(const int64_t* node_ptr, const int64_t* edge_ptr, const int32_t* store_edge_index,
                                int64_t store_num_edges, const uint8_t* pair_first, const int64_t* graph_ids, int64_t B,
                                int64_t full_nodes, const int32_t* roots, int64_t seed, int k, int l1, int l2, int whole_graph,
                                void* workspace, int64_t workspace_bytes, int64_t* offsets, void* stream);
PGNN_API int pgnn_extract_fill_chem(const int64_t* node_ptr, const int64_t* edge_ptr, const uint8_t* store_x,
                                    const int32_t* store_edge_index, int64_t store_num_edges, const uint8_t* store_edge_attr,
                                    const uint8_t* pair_first, const int64_t* graph_ids, int64_t B, int64_t full_nodes,
                                    const void* workspace, const int64_t* offsets, int64_t* x_substruct,
                                    int64_t* edge_index_substruct, int64_t* edge_attr_substruct, int64_t* center_substruct_idx,
                                    int64_t* x_context, int64_t* edge_index_context, int64_t* edge_attr_context,
                                    int64_t* overlap_context_substruct_idx, int64_t* batch_overlapped_context,
                                    int64_t* overlapped_context_size, void* stream);
PGNN_API int pgnn_extract_fill_bio(const int64_t* node_ptr, const int64_t* edge_ptr, const int32_t* store_edge_index,
                                   int64_t store_num_edges, const uint16_t* store_edge_bits, const uint8_t* pair_first,
                                   const int64_t* graph_ids, int64_t B, int64_t full_nodes, const void* workspace,
                                   const int64_t* offsets, float* x_context, int64_t* edge_index_context,
                                   float* edge_attr_context, int64_t* overlap_context_substruct_idx,
                                   int64_t* batch_overlapped_context, int64_t* overlapped_context_size, void* stream);

/* Multi-tensor Adam: torch.optim.Adam(model.parameters(), lr=args.lr, weight_decay=args.decay).step()
 * (chem/pretrain_masking.py:134-136,72-74; chem/pretrain_contextpred.py:160-161,96-97) for every tensor in one launch.
 * `chunks` is a DEVICE array; each chunk is a contiguous run of at most a few thousand elements of one tensor
 * (one CTA per chunk).  grad is read as grad*grad_scale (1/world_size folds the data-parallel mean in) and is not
 * modified.  Hyper-parameters are doubles (Python floats): 1-beta and the bias corrections are formed in double on the
 * host and rounded to fp32 once, as torch does.  step >= 1 is the 1-based step count.  legacy_eps = 0: current torch (denom = sqrt(v)/sqrt(bc2) + eps);
 * legacy_eps = 1: torch 1.0.1 as pinned by the reference (denom = sqrt(v) + eps, step = lr*sqrt(bc2)/bc1). */
typedef struct PgnnAdamChunk {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t n;
} PgnnAdamChunk;
PGNN_API int pgnn_adam_step(const PgnnAdamChunk* chunks, int64_t num_chunks, double lr, double beta1, double beta2, double eps,
                            double weight_decay, double grad_scale, int64_t step, int legacy_eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Gradient all-reduce over NVLink peer memory (SURVEY.md section 8(e)).  In place, two-shot (reduce-scatter by peer loads,
 * all-gather by peer stores, three flag barriers), bit-identical on every rank, no library collective.
 *   bufs  : DEVICE array of `world` pointers: the peer-mapped address of every rank's fp32 buffer of n elements (same offset
 *           of a symmetric allocation on every rank; bufs[rank] is the local one)
 *   flags : DEVICE array of `world` pointers to every rank's flag words (uint32[world], zero before the first call,
 *           used by these calls only)
 *   scratch: local device buffer of pgnn_allreduce_p2p_scratch_floats(n, world) floats
 *   epoch : 0, 1, 2, ... incremented by the caller on every call, identical on all ranks
 * On return (stream order) every rank's buffer holds scale * sum over ranks.  A rank that never arrives traps the waiting
 * kernels after ~60 s (sticky CUDA error) instead of hanging. */
PGNN_API int64_t pgnn_allreduce_p2p_scratch_floats(int64_t n, int world);
PGNN_API int pgnn_allreduce_p2p(void* const* bufs, void* const* flags, int rank, int world, int64_t n, float scale,
                                float* scratch, int64_t scratch_floats, int64_t epoch, void* stream);
/* One-kernel, OUT-OF-PLACE form (round 2): one launch, two flag exchanges instead of five launches and three barriers.
 *   in / out : DEVICE arrays of `world` peer-mapped pointers to every rank's input / output buffer (n floats each, distinct
 *              symmetric allocations); on return (stream order) out[rank] holds scale * sum over ranks of in[.], bit-identical
 *              on every rank (fixed summation order); the input buffers are left untouched and may be rewritten
 *   flags    : as above, but uint32[128] per rank: this entry uses words [64, 128)
 *   mc_in / mc_out : multicast mappings of the buffers (both non-null: multimem.ld_reduce / multimem.st, the NVSwitch sums and
 *              broadcasts; n % (4*world) == 0), else null
 *   counter  : LOCAL device uint32, zero before the first call */
PGNN_API int pgnn_allreduce_fused(void* const* in, void* const* out, void* const* flags, float* mc_in, float* mc_out,
                                  unsigned int* counter, int rank, int world, int64_t n, float scale, int64_t epoch, void* stream);
/* EXPERIMENTAL, not yet measured on hardware and not used by default: the same exchange with the NVSwitch doing the sum
 * (multimem.ld_reduce / multimem.st on the multicast mapping `mc_buf` of the symmetric buffer).  n % (4*world) == 0;
 * two flag barriers per call (own epoch counter; do not share a flag array with pgnn_allreduce_p2p). */
PGNN_API int pgnn_allreduce_nvls(float* mc_buf, void* const* flags, int rank, int world, int64_t n, float scale,
                                 int64_t epoch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PGNN_B200_H */
