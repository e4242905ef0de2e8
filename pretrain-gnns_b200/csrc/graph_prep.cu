// Graph preparation: stable bucketing of the COO edge list by target / by source, GCN degree
// normalisation and the per-node edge-feature summaries.  Integer results are bit-exact against
// oracle/graph_prep_oracle.py (stable argsort).
//
// Replaces the per-edge addressing that torch_geometric 1.0.3's MessagePassing.propagate performs for
// every layer (reference call sites chem/model.py:49,101,148,196; bio/model.py:52,111,163,218).
#include "common.cuh"

namespace {

// Bucketing kernels process up to TWO key arrays per launch (blockIdx.y selects the set): pgnn_graph_prep buckets the edge
// list by target and by source in the same four launches.  Keys outside [0, num_buckets) set PGNN_DEVERR_NODE_ID in the
// library's device error word and are dropped (the reference's index ops raise a device-side assert there).
struct BucketSet {
  const int64_t* keys;   // [n * stride]
  const int64_t* vals;   // optional payload copied in bucket order
  int* counts;           // [num_buckets + 1]; becomes the placement cursor after the scan
  int* tmp;              // [n]
  int* rowptr;           // [num_buckets + 1]
  int* order;            // [n]
  int* vals_out;         // [n] or null
  int64_t val_limit;     // > 0: payloads are indices too and must lie in [0, val_limit) (an edge's other endpoint)
};
struct BucketPair {
  BucketSet s[2];
};
__device__ __forceinline__ bool bucket_key_ok(const BucketSet& B, int64_t i, int64_t stride, int64_t val_stride, int64_t num_buckets, int64_t& k) {
  k = B.keys[i * stride];
  bool ok = k >= 0 && k < num_buckets;
  if (B.val_limit > 0) {
    const int64_t v = B.vals[i * val_stride];
    ok &= v >= 0 && v < B.val_limit;
  }
  return ok;
}

__global__ void k_histogram(const __grid_constant__ BucketPair P, int64_t stride, int64_t val_stride, int64_t n, int64_t num_buckets, unsigned int* __restrict__ err) {
  pdl_prologue();
  const BucketSet& B = P.s[blockIdx.y];
  bool bad = false;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t k;
    if (bucket_key_ok(B, i, stride, val_stride, num_buckets, k)) atomicAdd(&B.counts[k], 1);
    else bad = true;
  }
  if (bad && err) atomicOr(err, (unsigned)PGNN_DEVERR_NODE_ID);
}

// Exclusive scan of counts[0..n) into rowptr[0..n] (rowptr[n] = total) and, in place, into counts (the placement cursor).
// One CTA of 1024 threads per key set.  Each thread owns a CONTIGUOUS run of ceil(n / 1024) elements: it sums its run, the CTA
// scans the 1024 run totals once (two shuffle scans + one barrier pair), and the thread rewrites its run — one pass with a
// single block-wide synchronisation instead of one per 1024-element tile (node counts are 6 k - 32 k here: 6 - 32 tiles).
__global__ void __launch_bounds__(1024) k_exclusive_scan(const __grid_constant__ BucketPair P, int64_t n) {
  pdl_prologue();
  int* counts = P.s[blockIdx.x].counts;
  int* rowptr = P.s[blockIdx.x].rowptr;
  __shared__ int warp_tot[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t per = (n + 1023) / 1024;
  const int64_t lo = (int64_t)threadIdx.x * per, hi = (lo + per < n) ? lo + per : n;
  int mine = 0;
  for (int64_t i = lo; i < hi; ++i) mine += counts[i];
  int inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = warp_tot[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += t;
    }
    warp_tot[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  int run = (wid ? warp_tot[wid - 1] : 0) + inc - mine;  // exclusive prefix of this thread's run
  for (int64_t i = lo; i < hi; ++i) {
    const int v = counts[i];
    rowptr[i] = run;
    counts[i] = run;
    run += v;
  }
  if (threadIdx.x == 1023) rowptr[n] = warp_tot[31];
}

__global__ void k_place(const __grid_constant__ BucketPair P, int64_t stride, int64_t val_stride, int64_t n, int64_t num_buckets) {
  pdl_prologue();
  const BucketSet& B = P.s[blockIdx.y];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t k;
    if (!bucket_key_ok(B, i, stride, val_stride, num_buckets, k)) continue;  // flagged by k_histogram
    int pos = atomicAdd(&B.counts[k], 1);
    B.tmp[pos] = (int)i;
  }
}

// The atomic placement leaves every bucket holding the right SET in arbitrary order; rank each element
// among its bucket-mates by original position to obtain the stable order (rank by counting: bucket sizes
// are in-degrees / graph sizes / vocabulary hits, so the quadratic term stays tiny).
__global__ void k_rank_in_bucket(const __grid_constant__ BucketPair P, int64_t stride, int64_t val_stride, int64_t num_buckets) {
  pdl_prologue();
  const BucketSet& B = P.s[blockIdx.y];
  const int64_t placed = B.rowptr[num_buckets];  // == n unless out-of-range keys were dropped
  for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < placed; p += (int64_t)gridDim.x * blockDim.x) {
    const int me = B.tmp[p];
    const int64_t b = B.keys[(int64_t)me * stride];
    const int lo = B.rowptr[b], hi = B.rowptr[b + 1];
    int rank = 0;
    for (int q = lo; q < hi; ++q) rank += (B.tmp[q] < me);
    B.order[lo + rank] = me;
    if (B.vals_out) B.vals_out[lo + rank] = (int)B.vals[(int64_t)me * val_stride];
  }
}

__global__ void k_gcn_dinv(const int* __restrict__ rowptr, int64_t n, float* __restrict__ dinv) {
  pdl_prologue();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    // deg.pow(-0.5) over the loop-augmented edges: in-degree + 1 >= 1, never inf (chem/model.py:78-80).  Taken in fp64 and
    // rounded once: the fp32 reciprocal of an fp32 square root rounds twice and lands up to 1.3 ulp from the true value.
    const double deg = (double)(rowptr[i + 1] - rowptr[i] + 1);
    dinv[i] = (float)(1.0 / sqrt(deg));
  }
}

__global__ void k_chem_edge_summary(const int64_t* __restrict__ edge_attr, const int* __restrict__ rowptr,
                                    const int* __restrict__ nbr, const int* __restrict__ eid, int64_t n, int mode,
                                    const float* __restrict__ dinv, float* __restrict__ S, unsigned int* __restrict__ err) {
  pdl_prologue();
  bool bad = false;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float s[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) s[q] = 0.f;
    const int lo = rowptr[i], hi = rowptr[i + 1];
    for (int k = lo; k < hi; ++k) {
      const int64_t e = eid[k];
      const int64_t b0 = edge_attr[2 * e], b1 = edge_attr[2 * e + 1];
      bad |= (b0 < 0) | (b0 >= 6) | (b1 < 0) | (b1 >= 3);  // nn.Embedding(6, .) / (3, .) would raise (chem/model.py:30-31)
      const int a0 = (int)b0, a1 = (int)b1;
      const float w = agg_weight(mode, dinv, (int)i, nbr[k], hi - lo);
#pragma unroll
      for (int q = 0; q < 6; ++q) s[q] += (a0 == q) ? w : 0.f;
#pragma unroll
      for (int q = 0; q < 3; ++q) s[6 + q] += (a1 == q) ? w : 0.f;
    }
    const float wl = agg_weight(mode, dinv, (int)i, (int)i, hi - lo);
    s[4] += wl;  // self-loop: bond type 4, direction 0 (chem/model.py:42-45)
    s[6] += wl;
#pragma unroll
    for (int q = 0; q < 9; ++q) S[i * 9 + q] = s[q];
  }
  if (bad && err) atomicOr(err, (unsigned)PGNN_DEVERR_BOND_CODE);
}

__global__ void k_bio_edge_summary(const float* __restrict__ edge_attr, const int* __restrict__ rowptr,
                                   const int* __restrict__ nbr, const int* __restrict__ eid, int64_t n, int mode,
                                   const float* __restrict__ dinv, float* __restrict__ S) {
  pdl_prologue();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float s[10];
#pragma unroll
    for (int q = 0; q < 10; ++q) s[q] = 0.f;
    const int lo = rowptr[i], hi = rowptr[i + 1];
    for (int k = lo; k < hi; ++k) {
      const float* a = edge_attr + (int64_t)eid[k] * 9;
      const float w = agg_weight(mode, dinv, (int)i, nbr[k], hi - lo);
#pragma unroll
      for (int q = 0; q < 9; ++q) s[q] += w * a[q];
      s[9] += w;
    }
    const float wl = agg_weight(mode, dinv, (int)i, (int)i, hi - lo);
    s[7] += wl;  // self-loop row is one-hot at column 7 (bio/model.py:42-43)
    s[9] += wl;
#pragma unroll
    for (int q = 0; q < 10; ++q) S[i * 10 + q] = s[q];
  }
}

inline int grid_for(int64_t n, int threads) {
  int64_t b = ceil_div(n, threads);
  int64_t cap = (int64_t)kNumSMs * 8;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

}  // namespace

extern "C" {

int64_t pgnn_bucket_workspace_bytes(int64_t num_keys, int64_t num_buckets) {
  if (num_keys < 0 || num_buckets < 0) return PGNN_EINVAL;
  return align_up((num_buckets + 1) * 4, 256) + align_up((num_keys > 0 ? num_keys : 1) * 4, 256);
}

}  // extern "C"

namespace {
// one or two bucketings (sets) of `num_keys` keys into `num_buckets` buckets in four launches
int bucket_sets(BucketPair P, int nsets, int64_t key_stride, int64_t val_stride, int64_t num_keys, int64_t num_buckets, cudaStream_t st) {
  for (int k = 0; k < nsets; ++k) PGNN_CUDA(cudaMemsetAsync(P.s[k].counts, 0, (num_buckets + 1) * 4, st));
  unsigned int* err = pgnn_error_flag_ptr();
  const dim3 grid((unsigned)grid_for(num_keys, 256), (unsigned)nsets);
  if (num_keys > 0) {
    PGNN_CUDA(pgnn_launch(k_histogram, grid, dim3(256), 0, st, P, key_stride, val_stride, num_keys, num_buckets, err));
    PGNN_LAUNCH_CHECK();
  }
  PGNN_CUDA(pgnn_launch(k_exclusive_scan, dim3((unsigned)nsets), dim3(1024), 0, st, P, num_buckets));
  PGNN_LAUNCH_CHECK();
  if (num_keys > 0) {
    PGNN_CUDA(pgnn_launch(k_place, grid, dim3(256), 0, st, P, key_stride, val_stride, num_keys, num_buckets));
    PGNN_LAUNCH_CHECK();
    PGNN_CUDA(pgnn_launch(k_rank_in_bucket, grid, dim3(256), 0, st, P, key_stride, val_stride, num_buckets));
    PGNN_LAUNCH_CHECK();
  }
  return PGNN_OK;
}
}  // namespace

extern "C" {

int pgnn_bucket(const int64_t* keys, int64_t key_stride, int64_t num_keys, int64_t num_buckets, const int64_t* vals,
                int64_t val_stride, int32_t* rowptr, int32_t* order, int32_t* vals_out, void* workspace,
                int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(num_keys >= 0 && num_buckets >= 0 && rowptr && workspace);
  PGNN_CHECK_ARG(num_keys == 0 || (keys && order));
  PGNN_CHECK_ARG((vals == nullptr) == (vals_out == nullptr) || num_keys == 0);
  PGNN_CHECK_ARG(num_keys < (int64_t)1 << 31 && num_buckets < (int64_t)1 << 31);
  if (workspace_bytes < pgnn_bucket_workspace_bytes(num_keys, num_buckets)) return PGNN_EWORKSPACE;
  BucketPair P = {};
  P.s[0].keys = keys; P.s[0].vals = vals;
  P.s[0].counts = reinterpret_cast<int*>(workspace);
  P.s[0].tmp = reinterpret_cast<int*>(reinterpret_cast<char*>(workspace) + align_up((num_buckets + 1) * 4, 256));
  P.s[0].rowptr = rowptr; P.s[0].order = order; P.s[0].vals_out = vals_out;
  return bucket_sets(P, 1, key_stride, val_stride, num_keys, num_buckets, as_stream(stream));
}

int64_t pgnn_graph_prep_workspace_bytes(int64_t num_nodes, int64_t num_edges) {
  const int64_t one = pgnn_bucket_workspace_bytes(num_edges, num_nodes);
  return one < 0 ? one : 2 * one;
}

int pgnn_graph_prep(const int64_t* edge_index, int64_t num_edges, int64_t num_nodes, int32_t* rowptr_t,
                    int32_t* nbr_t, int32_t* eid_t, int32_t* rowptr_s, int32_t* nbr_s, int32_t* eid_s, void* workspace,
                    int64_t workspace_bytes, void* stream) {
  PGNN_CHECK_ARG(num_edges >= 0 && num_nodes >= 0 && rowptr_t && rowptr_s && workspace);
  PGNN_CHECK_ARG(num_edges == 0 || (edge_index && nbr_t && eid_t && nbr_s && eid_s));
  PGNN_CHECK_ARG(num_edges < (int64_t)1 << 31 && num_nodes < (int64_t)1 << 31);
  if (workspace_bytes < pgnn_graph_prep_workspace_bytes(num_nodes, num_edges)) return PGNN_EWORKSPACE;
  const int64_t* tgt = edge_index;
  const int64_t* src = edge_index ? edge_index + num_edges : nullptr;
  const int64_t one = pgnn_bucket_workspace_bytes(num_edges, num_nodes);
  BucketPair P = {};
  for (int k = 0; k < 2; ++k) {
    char* base = reinterpret_cast<char*>(workspace) + k * one;
    P.s[k].counts = reinterpret_cast<int*>(base);
    P.s[k].tmp = reinterpret_cast<int*>(base + align_up((num_nodes + 1) * 4, 256));
  }
  // set 0: bucket by target (edge_index[0]), payload = source; set 1: by source, payload = target (transpose graph)
  P.s[0].keys = tgt; P.s[0].vals = src; P.s[0].rowptr = rowptr_t; P.s[0].order = eid_t; P.s[0].vals_out = nbr_t;
  P.s[1].keys = src; P.s[1].vals = tgt; P.s[1].rowptr = rowptr_s; P.s[1].order = eid_s; P.s[1].vals_out = nbr_s;
  P.s[0].val_limit = P.s[1].val_limit = num_nodes;  // an edge with EITHER endpoint out of range is dropped from both bucketings
  return bucket_sets(P, 2, 1, 1, num_edges, num_nodes, as_stream(stream));
}

int pgnn_gcn_dinv(const int32_t* rowptr_t, int64_t num_nodes, float* dinv, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && (num_nodes == 0 || (rowptr_t && dinv)));
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CUDA(pgnn_launch(k_gcn_dinv, dim3(grid_for(num_nodes, 256)), dim3(256), 0, as_stream(stream), rowptr_t, num_nodes, dinv));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_chem_edge_summary(const int64_t* edge_attr, const int32_t* rowptr_t, const int32_t* nbr_t, const int32_t* eid_t,
                           int64_t num_nodes, int mode, const float* dinv, float* S, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && mode >= 0 && mode <= 2 && (mode != PGNN_AGG_GCN || dinv));
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(rowptr_t && S);
  PGNN_CUDA(pgnn_launch(k_chem_edge_summary, dim3(grid_for(num_nodes, 128)), dim3(128), 0, as_stream(stream), edge_attr, rowptr_t, nbr_t, eid_t, num_nodes,
                                                                               mode, dinv, S, pgnn_error_flag_ptr()));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_bio_edge_summary(const float* edge_attr, const int32_t* rowptr_t, const int32_t* nbr_t, const int32_t* eid_t,
                          int64_t num_nodes, int mode, const float* dinv, float* S, void* stream) {
  PGNN_CHECK_ARG(num_nodes >= 0 && mode >= 0 && mode <= 2 && (mode != PGNN_AGG_GCN || dinv));
  if (num_nodes == 0) return PGNN_OK;
  PGNN_CHECK_ARG(rowptr_t && S);
  PGNN_CUDA(pgnn_launch(k_bio_edge_summary, dim3(grid_for(num_nodes, 128)), dim3(128), 0, as_stream(stream), edge_attr, rowptr_t, nbr_t, eid_t, num_nodes,
                                                                              mode, dinv, S));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

}  // extern "C"
