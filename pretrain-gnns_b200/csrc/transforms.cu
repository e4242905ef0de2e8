// On-the-fly transforms and the remaining collators, on the device (SURVEY.md section 8(f), rows f4 and f1):
//
//   pgnn_mask_atoms        MaskAtom.__call__ with mask_edge=False (chem/util.py:189-241), applied to a collated batch:
//                          per graph int(n * mask_rate + 1) DISTINCT atoms drawn uniformly, their (type, chirality) saved as
//                          mask_node_label, their x row overwritten with [num_atom_type, 0].  The reference draws with
//                          Python's random.sample in a DataLoader worker; bit parity with that RNG is impossible, so the
//                          draw is defined here: node i of graph g gets the 64-bit key splitmix64(seed, position in the
//                          batch) and the k smallest keys of the graph are masked (a uniform k-subset).  Output order:
//                          ascending node index (the reference's is the arbitrary sample order; every consumer is a
//                          row gather + mean, so only the set matters).
//   pgnn_collate_lists     the per-graph index lists a batch carries next to its tensors, each entry offset by the running
//                          node count of its graph: masked_atom_indices (chem/batch.py:41-42), center_substruct_idx /
//                          overlap_context_substruct_idx with batch_overlapped_context and overlapped_context_size
//                          (chem/batch.py:170-199), center_node_idx (bio/batch.py:39-40).
//   pgnn_collate_bio       BatchFinetune / BatchMasking.from_data_list of bio/batch.py:17-50 for PPI ego graphs held in HBM:
//                          x float [N,1], edge_index int64 [2,E] + node offset, edge_attr float [E,9] from 9 packed bits,
//                          batch [N].
// All integer work, bit-exact against oracle/step_io_oracle.py.
#include "common.cuh"

namespace {

__device__ __forceinline__ int64_t mask_count(int64_t n, double rate) { return n > 0 ? (int64_t)((double)n * rate + 1.0) : 0; }

// mask_off[0..B] = exclusive scan of the per-graph sample sizes (one CTA, any B; B is a few hundred)
__global__ void __launch_bounds__(1024)
k_mask_scan(const int64_t* __restrict__ node_off, int64_t B, double rate, int64_t* __restrict__ mask_off) {
  pdl_prologue();
  __shared__ int64_t wsum[32];
  __shared__ int64_t carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < B; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    int64_t k = 0;
    if (i < B) {
      const int64_t n = node_off[i + 1] - node_off[i];
      k = mask_count(n, rate);
      if (k > n) k = n;
    }
    int64_t s = k;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (lane == 31) wsum[warp] = s;
    __syncthreads();
    if (warp == 0) {
      int64_t a = wsum[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int64_t t = __shfl_up_sync(0xffffffffu, a, d);
        if (lane >= d) a += t;
      }
      wsum[lane] = a;
    }
    __syncthreads();
    const int64_t pre = carry + (warp ? wsum[warp - 1] : 0);
    if (i < B) mask_off[i] = pre + s - k;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = pre + s;
    __syncthreads();
  }
  if (threadIdx.x == 0) mask_off[B] = carry;
}

// one warp per graph: rank every node's key among the graph's keys (ties by index), mask the k smallest
__global__ void __launch_bounds__(256)
k_mask_atoms(int64_t* __restrict__ x, const int64_t* __restrict__ node_off, int64_t B, double rate, int64_t mask_token, uint64_t seed,
             const int64_t* __restrict__ mask_off, int64_t* __restrict__ masked_idx, int64_t* __restrict__ labels) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t g = wid; g < B; g += nw) {
    const int64_t n0 = node_off[g], n = node_off[g + 1] - n0;
    int64_t k = mask_count(n, rate);
    if (k > n) k = n;
    int64_t out = mask_off[g];
    for (int64_t base = 0; base < n; base += 32) {
      const int64_t i = base + lane;
      bool sel = false;
      if (i < n) {
        const uint64_t ki = splitmix64(seed, (uint64_t)(n0 + i));
        int64_t rank = 0;
        for (int64_t j = 0; j < n; ++j) {
          const uint64_t kj = splitmix64(seed, (uint64_t)(n0 + j));
          rank += (kj < ki) || (kj == ki && j < i);
        }
        sel = rank < k;
      }
      const unsigned m = __ballot_sync(0xffffffffu, sel);
      if (sel) {
        const int64_t pos = out + __popc(m & ((1u << lane) - 1u));
        const int64_t gid = n0 + i;
        masked_idx[pos] = gid;
        labels[2 * pos] = x[2 * gid];
        labels[2 * pos + 1] = x[2 * gid + 1];
        x[2 * gid] = mask_token;      // chem/util.py:241: data.x[atom_idx] = [num_atom_type, 0]
        x[2 * gid + 1] = 0;
      }
      out += __popc(m);
    }
  }
}

// ragged per-graph lists: out[list_off[i] + j] = values[ptr[g] + j] + add[i]; seg[...] = i; sizes[i] = length
__global__ void __launch_bounds__(1024)
k_list_scan(const int64_t* __restrict__ ptr, const int64_t* __restrict__ ids, int64_t B, int64_t* __restrict__ list_off) {
  pdl_prologue();
  __shared__ int64_t wsum[32];
  __shared__ int64_t carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < B; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    int64_t k = 0;
    if (i < B) k = ptr[ids[i] + 1] - ptr[ids[i]];
    int64_t s = k;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (lane == 31) wsum[warp] = s;
    __syncthreads();
    if (warp == 0) {
      int64_t a = wsum[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int64_t t = __shfl_up_sync(0xffffffffu, a, d);
        if (lane >= d) a += t;
      }
      wsum[lane] = a;
    }
    __syncthreads();
    const int64_t pre = carry + (warp ? wsum[warp - 1] : 0);
    if (i < B) list_off[i] = pre + s - k;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = pre + s;
    __syncthreads();
  }
  if (threadIdx.x == 0) list_off[B] = carry;
}

__global__ void __launch_bounds__(256)
k_list_fill(const int64_t* __restrict__ ptr, const int32_t* __restrict__ values, const int64_t* __restrict__ ids, int64_t B,
            const int64_t* __restrict__ add, const int64_t* __restrict__ list_off, int64_t* __restrict__ out, int64_t* __restrict__ seg,
            int64_t* __restrict__ sizes) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = wid; i < B; i += nw) {
    const int64_t g = ids[i], p0 = ptr[g], len = ptr[g + 1] - p0, o = list_off[i], a = add ? add[i] : 0;
    for (int64_t j = lane; j < len; j += 32) {
      out[o + j] = (int64_t)values[p0 + j] + a;
      if (seg) seg[o + j] = i;
    }
    if (sizes && lane == 0) sizes[i] = len;
  }
}

// bio graphs: x is the constant dummy label 1.0 (bio/loader.py:47), edge attributes are 9 bits (bio/loader.py:57-75)
__global__ void __launch_bounds__(256)
k_collate_bio_fill(const int64_t* __restrict__ node_ptr, const int64_t* __restrict__ edge_ptr, const int32_t* __restrict__ sei,
                   int64_t store_edges, const uint16_t* __restrict__ sbits, const int64_t* __restrict__ ids, int64_t B,
                   const int64_t* __restrict__ node_off, const int64_t* __restrict__ edge_off, float* __restrict__ x,
                   int64_t* __restrict__ edge_index, float* __restrict__ edge_attr, int64_t* __restrict__ batch) {
  pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nw = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t E = edge_off[B];
  for (int64_t i = wid; i < B; i += nw) {
    const int64_t g = ids[i];
    const int64_t n = node_ptr[g + 1] - node_ptr[g], e0 = edge_ptr[g], e = edge_ptr[g + 1] - e0;
    const int64_t no = node_off[i], eo = edge_off[i];
    for (int64_t k = lane; k < n; k += 32) {
      x[no + k] = 1.f;
      batch[no + k] = i;
    }
    for (int64_t k = lane; k < e; k += 32) {
      edge_index[eo + k] = no + sei[e0 + k];
      edge_index[E + eo + k] = no + sei[store_edges + e0 + k];
      const unsigned bits = sbits[e0 + k];
#pragma unroll
      for (int q = 0; q < 9; ++q) edge_attr[(eo + k) * 9 + q] = (bits >> q) & 1u ? 1.f : 0.f;
    }
  }
}

// same scan as chem's collate (node and edge counts of the selected graphs)
__global__ void __launch_bounds__(1024)
k_collate_scan2(const int64_t* __restrict__ node_ptr, const int64_t* __restrict__ edge_ptr, const int64_t* __restrict__ ids, int64_t B,
                int64_t* __restrict__ node_off, int64_t* __restrict__ edge_off) {
  pdl_prologue();
  __shared__ int64_t wn[32], we[32];
  __shared__ int64_t carry_n, carry_e;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_n = carry_e = 0;
  __syncthreads();
  for (int64_t base = 0; base < B; base += blockDim.x) {
    const int64_t i = base + threadIdx.x;
    int64_t n = 0, e = 0;
    if (i < B) {
      const int64_t g = ids[i];
      n = node_ptr[g + 1] - node_ptr[g];
      e = edge_ptr[g + 1] - edge_ptr[g];
    }
    int64_t sn = n, se = e;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t tn = __shfl_up_sync(0xffffffffu, sn, d), te = __shfl_up_sync(0xffffffffu, se, d);
      if (lane >= d) { sn += tn; se += te; }
    }
    if (lane == 31) { wn[warp] = sn; we[warp] = se; }
    __syncthreads();
    if (warp == 0) {
      int64_t a = wn[lane], b = we[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int64_t ta = __shfl_up_sync(0xffffffffu, a, d), tb = __shfl_up_sync(0xffffffffu, b, d);
        if (lane >= d) { a += ta; b += tb; }
      }
      wn[lane] = a; we[lane] = b;
    }
    __syncthreads();
    const int64_t pn = carry_n + (warp ? wn[warp - 1] : 0), pe = carry_e + (warp ? we[warp - 1] : 0);
    if (i < B) { node_off[i] = pn + sn - n; edge_off[i] = pe + se - e; }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) { carry_n = pn + sn; carry_e = pe + se; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { node_off[B] = carry_n; edge_off[B] = carry_e; }
}

inline unsigned warp_grid(int64_t items) {
  const int64_t blocks = ceil_div(items, 8);
  return (unsigned)(blocks < 1 ? 1 : (blocks < 8 * kNumSMs ? blocks : 8 * kNumSMs));
}

}  // namespace

extern "C" {

int64_t pgnn_mask_atoms_count(const int64_t* node_off_host, int64_t B, double mask_rate) {
  if (!node_off_host || B < 0) return PGNN_EINVAL;
  int64_t m = 0;
  for (int64_t g = 0; g < B; ++g) {
    const int64_t n = node_off_host[g + 1] - node_off_host[g];
    int64_t k = n > 0 ? (int64_t)((double)n * mask_rate + 1.0) : 0;  // int(num_atoms * mask_rate + 1), chem/util.py:229
    m += k > n ? n : k;
  }
  return m;
}

int pgnn_mask_atoms(int64_t* x, const int64_t* node_off, int64_t B, double mask_rate, int64_t mask_token, int64_t seed,
                    int64_t* mask_off, int64_t* masked_atom_indices, int64_t* mask_node_label, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && mask_rate >= 0.0 && node_off && mask_off);
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(pgnn_launch(k_mask_scan, dim3(1), dim3(1024), 0, st, node_off, B, mask_rate, mask_off));
  PGNN_LAUNCH_CHECK();
  if (B == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && masked_atom_indices && mask_node_label);
  PGNN_CUDA(pgnn_launch(k_mask_atoms, dim3(warp_grid(B)), dim3(256), 0, st, x, node_off, B, mask_rate, mask_token, (uint64_t)seed,
                        (const int64_t*)mask_off, masked_atom_indices, mask_node_label));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_collate_lists(const int64_t* list_ptr, const int32_t* values, const int64_t* graph_ids, int64_t B, const int64_t* add_per_graph,
                       int64_t* list_off, int64_t* out, int64_t* seg, int64_t* sizes, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && list_ptr && list_off);
  cudaStream_t st = as_stream(stream);
  PGNN_CHECK_ARG(B == 0 || graph_ids);
  PGNN_CUDA(pgnn_launch(k_list_scan, dim3(1), dim3(1024), 0, st, list_ptr, graph_ids, B, list_off));
  PGNN_LAUNCH_CHECK();
  if (B == 0) return PGNN_OK;
  PGNN_CHECK_ARG(values && out);
  PGNN_CUDA(pgnn_launch(k_list_fill, dim3(warp_grid(B)), dim3(256), 0, st, list_ptr, values, graph_ids, B, add_per_graph, (const int64_t*)list_off, out,
                        seg, sizes));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_collate_bio(const int64_t* node_ptr, const int64_t* edge_ptr, const int32_t* store_edge_index, int64_t store_num_edges,
                     const uint16_t* store_edge_bits, const int64_t* graph_ids, int64_t B, int64_t* node_off, int64_t* edge_off, float* x,
                     int64_t* edge_index, float* edge_attr, int64_t* batch, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && store_num_edges >= 0 && node_ptr && edge_ptr && node_off && edge_off);
  if (B > 0) PGNN_CHECK_ARG(graph_ids && x && batch);
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(pgnn_launch(k_collate_scan2, dim3(1), dim3(1024), 0, st, node_ptr, edge_ptr, graph_ids, B, node_off, edge_off));
  PGNN_LAUNCH_CHECK();
  if (B == 0) return PGNN_OK;
  PGNN_CUDA(pgnn_launch(k_collate_bio_fill, dim3(warp_grid(B)), dim3(256), 0, st, node_ptr, edge_ptr, store_edge_index, store_num_edges, store_edge_bits,
                        graph_ids, B, (const int64_t*)node_off, (const int64_t*)edge_off, x, edge_index, edge_attr, batch));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

}  // extern "C"
