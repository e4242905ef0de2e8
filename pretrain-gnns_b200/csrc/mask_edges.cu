// Edge masking transforms on a collated batch, on the device (SURVEY.md section 8(f), row f4):
//
//   pgnn_mask_edges_chem   the mask_edge=True half of MaskAtom.__call__ (chem/util.py:243-272) + BatchMasking's offsets
//                          (chem/batch.py:40-42).  Per graph: L = the edge columns with an endpoint among the masked atoms, in
//                          ascending column order (the reference's double loop appends each bond index once, in order);
//                          connected_edge_indices = L[::2] (one column per bond when the two directions are adjacent),
//                          mask_edge_label = edge_attr[L[::2]] read BEFORE the overwrite, edge_attr[L] = [num_edge_type, 0].
//                          The rule is applied literally (rank of a column inside L, every second one), so inputs that are not
//                          paired get exactly what the reference's code would give them.
//   pgnn_mask_edges_bio    MaskEdge.__call__ (bio/util.py:46-104) + bio BatchMasking's offsets (bio/batch.py:93-96).  Per graph
//                          of e/2 bond pairs: int(e/2 * mask_rate + 1) DISTINCT pairs drawn uniformly (the k smallest
//                          splitmix64(seed, column id) keys: a uniform k-subset; the reference's random.sample cannot be matched
//                          bit for bit), masked_edge_idx = the pairs' first columns (2i + edge offset, ascending),
//                          mask_edge_label = their attribute rows, then both directions set to [0,0,0,0,0,0,0,0,1].
// Integer / 0-1 float work, bit-exact against oracle/step_io_oracle.py (mask_edges_chem, mask_edges_bio).
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kKeyCache = 4096;  // pairs whose keys fit the CTA's shared memory (32 KB); larger graphs recompute keys

__device__ __forceinline__ int64_t edge_mask_count(int64_t pairs, double rate) {
  if (pairs <= 0) return 0;
  const int64_t k = (int64_t)((double)pairs * rate + 1.0);  // int(num_edges * mask_rate + 1), bio/util.py:80
  return k > pairs ? pairs : k;
}

__device__ __forceinline__ int block_scan1(bool a, int* sh, int& t) { return block_scan_flag<kWarps>(a, sh, t); }

__global__ void __launch_bounds__(256)
k_flag_nodes(const int64_t* __restrict__ idx, int64_t M, int64_t N, uint8_t* __restrict__ flags, unsigned int* __restrict__ err) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int64_t v = idx[i];
  if (v < 0 || v >= N) {
    if (err) atomicOr(err, PGNN_DEVERR_GATHER);
    return;
  }
  flags[v] = 1;
}

__device__ __forceinline__ bool connected(const int64_t* __restrict__ ei, int64_t E, int64_t N, const uint8_t* __restrict__ flags, int64_t j) {
  const int64_t u = ei[j], v = ei[E + j];
  return ((uint64_t)u < (uint64_t)N && flags[u]) || ((uint64_t)v < (uint64_t)N && flags[v]);
}

// counts[g] = ceil(|L_g| / 2)
__global__ void __launch_bounds__(kThreads)
k_mask_edges_chem_count(const int64_t* __restrict__ ei, int64_t E, int64_t N, const int64_t* __restrict__ edge_off, const uint8_t* __restrict__ flags,
                        int64_t* __restrict__ counts) {
  pdl_prologue();
  __shared__ int sh[kWarps];
  const int64_t g = blockIdx.x, e0 = edge_off[g], e = edge_off[g + 1] - e0;
  int total = 0;
  for (int64_t base = 0; base < e; base += kThreads) {
    const int64_t j = base + threadIdx.x;
    int t;
    block_scan1(j < e && connected(ei, E, N, flags, e0 + j), sh, t);
    total += t;
  }
  if (threadIdx.x == 0) counts[g] = (total + 1) / 2;
}

__global__ void __launch_bounds__(32)
k_scan_counts(const int64_t* __restrict__ counts, int64_t B, int64_t* __restrict__ off) {
  pdl_prologue();
  warp_scan_to(B, off, [&](int64_t i) { return counts[i]; });
}

__global__ void __launch_bounds__(kThreads)
k_mask_edges_chem_fill(const int64_t* __restrict__ ei, int64_t E, int64_t N, const int64_t* __restrict__ edge_off, const uint8_t* __restrict__ flags,
                       const int64_t* __restrict__ conn_off, int64_t mask_token, int64_t* __restrict__ edge_attr, int64_t* __restrict__ conn,
                       int64_t* __restrict__ labels) {
  pdl_prologue();
  __shared__ int sh[kWarps];
  const int64_t g = blockIdx.x, e0 = edge_off[g], e = edge_off[g + 1] - e0, o = conn_off[g];
  int carry = 0;
  for (int64_t base = 0; base < e; base += kThreads) {
    const int64_t j = base + threadIdx.x;
    const bool f = j < e && connected(ei, E, N, flags, e0 + j);
    int t;
    const int r = carry + block_scan1(f, sh, t);   // rank of this column inside L
    if (f) {
      const int64_t col = e0 + j;
      if ((r & 1) == 0) {                            // L[::2]
        conn[o + (r >> 1)] = col;                    // + cumsum_edge: chem/batch.py:41-42
        labels[2 * (o + (r >> 1))] = edge_attr[2 * col];
        labels[2 * (o + (r >> 1)) + 1] = edge_attr[2 * col + 1];
      }
      edge_attr[2 * col] = mask_token;               // chem/util.py:263-265
      edge_attr[2 * col + 1] = 0;
    }
    carry += t;
  }
}

__global__ void __launch_bounds__(32)
k_mask_edges_bio_scan(const int64_t* __restrict__ edge_off, int64_t B, double rate, int64_t* __restrict__ mask_off) {
  pdl_prologue();
  warp_scan_to(B, mask_off, [&](int64_t i) { return edge_mask_count((edge_off[i + 1] - edge_off[i]) >> 1, rate); });
}

__global__ void __launch_bounds__(kThreads)
k_mask_edges_bio(float* __restrict__ edge_attr, const int64_t* __restrict__ edge_off, double rate, uint64_t seed, const int64_t* __restrict__ mask_off,
                 int64_t* __restrict__ masked_idx, float* __restrict__ labels) {
  pdl_prologue();
  __shared__ uint64_t keys[kKeyCache];
  __shared__ int sh[kWarps];
  const int64_t g = blockIdx.x, e0 = edge_off[g];
  const int64_t m = (edge_off[g + 1] - e0) >> 1;
  const int64_t k = edge_mask_count(m, rate), o = mask_off[g];
  const bool cached = m <= kKeyCache;
  if (cached)
    for (int64_t i = threadIdx.x; i < m; i += kThreads) keys[i] = splitmix64(seed, (uint64_t)(e0 + 2 * i));
  __syncthreads();
  int carry = 0;
  for (int64_t base = 0; base < m; base += kThreads) {
    const int64_t i = base + threadIdx.x;
    bool sel = false;
    if (i < m) {
      const uint64_t ki = cached ? keys[i] : splitmix64(seed, (uint64_t)(e0 + 2 * i));
      int64_t rank = 0;
      for (int64_t j = 0; j < m && rank < k; ++j) {
        const uint64_t kj = cached ? keys[j] : splitmix64(seed, (uint64_t)(e0 + 2 * j));
        rank += (kj < ki) || (kj == ki && j < i);
      }
      sel = rank < k;
    }
    int t;
    const int r = carry + block_scan1(sel, sh, t);
    if (sel) {
      const int64_t col = e0 + 2 * i;
      masked_idx[o + r] = col;                      // 2 * i + cumsum_edge: bio/util.py:83-84, bio/batch.py:95-96
#pragma unroll
      for (int q = 0; q < 9; ++q) {
        labels[(o + r) * 9 + q] = edge_attr[col * 9 + q];
        const float mv = q == 8 ? 1.f : 0.f;        // bio/util.py:98-102
        edge_attr[col * 9 + q] = mv;
        edge_attr[(col + 1) * 9 + q] = mv;
      }
    }
    carry += t;
  }
}

}  // namespace

extern "C" {

int64_t pgnn_mask_edges_chem_workspace_bytes(int64_t N, int64_t B) {
  if (N < 0 || B < 0) return PGNN_EINVAL;
  return align_up(N > 0 ? N : 1, 256) + align_up((B > 0 ? B : 1) * 8, 256);
}

int pgnn_mask_edges_chem(const int64_t* edge_index, int64_t* edge_attr, const int64_t* edge_off, int64_t B, int64_t N, int64_t E,
                         const int64_t* masked_atom_indices, int64_t M, int64_t num_edge_type, void* workspace, int64_t workspace_bytes,
                         int64_t* conn_off, int64_t* connected_edge_indices, int64_t* mask_edge_label, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && N >= 0 && E >= 0 && M >= 0 && edge_off && conn_off && workspace);
  if (workspace_bytes < pgnn_mask_edges_chem_workspace_bytes(N, B)) return PGNN_EWORKSPACE;
  cudaStream_t st = as_stream(stream);
  uint8_t* flags = reinterpret_cast<uint8_t*>(workspace);
  int64_t* counts = reinterpret_cast<int64_t*>(flags + align_up(N > 0 ? N : 1, 256));
  PGNN_CUDA(cudaMemsetAsync(flags, 0, (size_t)(N > 0 ? N : 1), st));
  if (M > 0) {
    PGNN_CHECK_ARG(masked_atom_indices);
    PGNN_CUDA(pgnn_launch(k_flag_nodes, dim3((unsigned)ceil_div(M, 256)), dim3(256), 0, st, masked_atom_indices, M, N, flags, pgnn_error_flag_ptr()));
    PGNN_LAUNCH_CHECK();
  }
  if (B > 0) {
    PGNN_CHECK_ARG(E == 0 || (edge_index && edge_attr));
    PGNN_CUDA(pgnn_launch(k_mask_edges_chem_count, dim3((unsigned)B), dim3(kThreads), 0, st, edge_index, E, N, edge_off, (const uint8_t*)flags, counts));
    PGNN_LAUNCH_CHECK();
  }
  PGNN_CUDA(pgnn_launch(k_scan_counts, dim3(1), dim3(32), 0, st, (const int64_t*)counts, B, conn_off));
  PGNN_LAUNCH_CHECK();
  if (B > 0) {
    PGNN_CHECK_ARG(connected_edge_indices && mask_edge_label);
    PGNN_CUDA(pgnn_launch(k_mask_edges_chem_fill, dim3((unsigned)B), dim3(kThreads), 0, st, edge_index, E, N, edge_off, (const uint8_t*)flags,
                          (const int64_t*)conn_off, num_edge_type, edge_attr, connected_edge_indices, mask_edge_label));
    PGNN_LAUNCH_CHECK();
  }
  return PGNN_OK;
}

int64_t pgnn_mask_edges_bio_count(const int64_t* edge_off_host, int64_t B, double mask_rate) {
  if (!edge_off_host || B < 0) return PGNN_EINVAL;
  int64_t m = 0;
  for (int64_t g = 0; g < B; ++g) {
    const int64_t pairs = (edge_off_host[g + 1] - edge_off_host[g]) >> 1;
    if (pairs <= 0) continue;
    const int64_t k = (int64_t)((double)pairs * mask_rate + 1.0);
    m += k > pairs ? pairs : k;
  }
  return m;
}

int pgnn_mask_edges_bio(float* edge_attr, const int64_t* edge_off, int64_t B, double mask_rate, int64_t seed, int64_t* mask_off,
                        int64_t* masked_edge_idx, float* mask_edge_label, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && mask_rate >= 0.0 && edge_off && mask_off);
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(pgnn_launch(k_mask_edges_bio_scan, dim3(1), dim3(32), 0, st, edge_off, B, mask_rate, mask_off));
  PGNN_LAUNCH_CHECK();
  if (B == 0) return PGNN_OK;
  PGNN_CHECK_ARG(edge_attr && masked_edge_idx && mask_edge_label);
  PGNN_CUDA(pgnn_launch(k_mask_edges_bio, dim3((unsigned)B), dim3(kThreads), 0, st, edge_attr, edge_off, mask_rate, (uint64_t)seed,
                        (const int64_t*)mask_off, masked_edge_idx, mask_edge_label));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

}  // extern "C"
