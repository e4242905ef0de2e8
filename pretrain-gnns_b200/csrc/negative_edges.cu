// NegativeEdge (chem/util.py:22-52, bio/util.py:16-44) on a collated batch, with BatchAE's offsets (chem/batch.py:69-121,
// bio/batch.py:123-175), on the device.
//
// The reference, per graph of n nodes and e directed columns (graph-local ids): draw C = randint(0, n, (2, 5e)); walk the
// candidates j = 0 .. 5e-1 in order and accept (a, b) = C[:, j] iff a != b, (a, b) is not a column of edge_index (a DIRECTED
// test: the reverse of a one-direction edge is a valid negative) and (a, b) was not accepted before; after each candidate stop
// when the accepted count == e / 2 (a Python-3 float comparison: an odd e never stops early, e = 0 draws nothing).  Output:
// the accepted columns in candidate order, plus the running node count (BatchAE.from_data_list).
//
// The draw is DEFINED here (torch.randint cannot be matched bit for bit): candidate j of the graph in batch slot g, whose
// columns start at e0 = edge_off[g], is
//     a = splitmix64(seed, 2 (5 e0 + j)) mod n,    b = splitmix64(seed, 2 (5 e0 + j) + 1) mod n
// (modulo bias below n / 2^64).  A graph with n = 0 draws nothing.  Bit-exact against tests/edgepred_oracle.py
// (negative_edge_candidates + negative_edge, the reference's loop restated literally) and synthetic.negative_edge_index.
//
// One CTA per graph takes the candidates in chunks of one CTA width.  The "forbidden" set (the graph's columns, then every
// accepted pair) is an n^2-bit bitmap in shared memory for n <= kSmemMaxN, else an open-addressing hash in global memory of
// kHashPerColumn slots per edge column (at most e + 5e keys: load <= 0.75).  Inside a chunk, duplicates of a pair keep only
// their earliest valid candidate (a small shared hash: key -> smallest thread index); a block scan ranks the survivors and the
// remaining quota cuts them.  Accepted pairs are staged at the graph's capacity offset, then packed into the [2, M] output.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunkSlots = 2 * kThreads;             // in-chunk dedup hash (<= kThreads keys: load <= 0.5)
constexpr int kBitmapBytes = 64 * 1024;               // dynamic shared memory of the bitmap path
constexpr int64_t kSmemMaxN = 724;                    // 724^2 bits <= kBitmapBytes * 8
constexpr int64_t kHashPerColumn = 8;
constexpr unsigned long long kEmpty = ~0ull;

__host__ __device__ __forceinline__ int64_t neg_capacity(int64_t e) { return e <= 0 ? 0 : (e & 1) ? 5 * e : e / 2; }

__device__ __forceinline__ uint64_t pair_key(uint32_t a, uint32_t b) { return ((uint64_t)a << 32) | b; }
__device__ __forceinline__ uint64_t hash_start(uint64_t key, uint64_t size) { return __umul64hi(splitmix64(0, key), size); }

// The forbidden set of one graph: a bitmap in shared memory or a global hash (volatile reads: other threads of the CTA insert
// between barriers).
struct Forbidden {
  uint32_t* bits;
  unsigned long long* slots;
  uint64_t n, size;
  bool smem;

  __device__ bool has(uint32_t a, uint32_t b) const {
    if (smem) {
      const uint64_t i = (uint64_t)a * n + b;
      return (bits[i >> 5] >> (i & 31)) & 1u;
    }
    const uint64_t key = pair_key(a, b);
    for (uint64_t s = hash_start(key, size);; s = s + 1 == size ? 0 : s + 1) {
      const unsigned long long k = reinterpret_cast<volatile unsigned long long*>(slots)[s];
      if (k == key) return true;
      if (k == kEmpty) return false;
    }
  }
  __device__ void add(uint32_t a, uint32_t b) {
    if (smem) {
      const uint64_t i = (uint64_t)a * n + b;
      atomicOr(&bits[i >> 5], 1u << (i & 31));
      return;
    }
    const uint64_t key = pair_key(a, b);
    for (uint64_t s = hash_start(key, size);; s = s + 1 == size ? 0 : s + 1) {
      const unsigned long long prev = atomicCAS(&slots[s], kEmpty, (unsigned long long)key);
      if (prev == kEmpty || prev == key) return;
    }
  }
};

__global__ void __launch_bounds__(32)
k_negative_capacity_scan(const int64_t* __restrict__ edge_off, int64_t B, int64_t* __restrict__ cap_off) {
  pdl_prologue();
  warp_scan_to(B, cap_off, [&](int64_t i) { return neg_capacity(edge_off[i + 1] - edge_off[i]); });
}

__global__ void __launch_bounds__(kThreads)
k_negative_select(const int64_t* __restrict__ ei, int64_t E, const int64_t* __restrict__ node_off, const int64_t* __restrict__ edge_off,
                  uint64_t seed, const int64_t* __restrict__ cap_off, int64_t capacity, unsigned long long* __restrict__ hash,
                  unsigned long long* __restrict__ staged, int64_t* __restrict__ counts, unsigned int* __restrict__ err) {
  pdl_prologue();
  extern __shared__ uint32_t bits[];
  __shared__ unsigned long long ckey[kChunkSlots];
  __shared__ int cmin[kChunkSlots];
  __shared__ int sh[kWarps];
  const int64_t g = blockIdx.x, n0 = node_off[g], n = node_off[g + 1] - n0, e0 = edge_off[g], e = edge_off[g + 1] - e0;
  const int64_t K = n > 0 && e > 0 ? 5 * e : 0;
  const int64_t quota = (e & 1) ? K : e / 2;   // an odd e never stops early: every valid candidate may be taken
  const int64_t o = cap_off[g];
  Forbidden F{bits, hash + kHashPerColumn * e0, (uint64_t)(n > 0 ? n : 0), (uint64_t)(kHashPerColumn * (e > 0 ? e : 0)), n <= kSmemMaxN};
  if (F.smem) {
    for (int64_t i = threadIdx.x; i < (int64_t)((F.n * F.n + 31) >> 5); i += kThreads) bits[i] = 0u;
  } else {
    for (int64_t i = threadIdx.x; i < (int64_t)F.size; i += kThreads) F.slots[i] = kEmpty;
  }
  for (int i = threadIdx.x; i < kChunkSlots; i += kThreads) ckey[i] = kEmpty, cmin[i] = kThreads;
  __syncthreads();
  bool bad = false;
  for (int64_t j = threadIdx.x; j < e; j += kThreads) {   // the graph's own columns; an endpoint outside the graph is ignored
    const int64_t u = ei[e0 + j] - n0, v = ei[E + e0 + j] - n0;
    if (u >= 0 && u < n && v >= 0 && v < n) F.add((uint32_t)u, (uint32_t)v);
    else bad = true;
  }
  if (bad && err) atomicOr(err, (unsigned)PGNN_DEVERR_GATHER);
  __syncthreads();
  int64_t taken = 0;
  for (int64_t base = 0; base < K && taken < quota; base += kThreads) {
    const int64_t j = base + threadIdx.x;
    uint32_t a = 0, b = 0;
    bool valid = false;
    if (j < K) {
      const uint64_t c = 2ull * (uint64_t)(5 * e0 + j);
      a = (uint32_t)(splitmix64(seed, c) % F.n);
      b = (uint32_t)(splitmix64(seed, c + 1) % F.n);
      valid = a != b && !F.has(a, b);
    }
    const uint64_t key = pair_key(a, b);
    int slot = 0;
    if (valid) {   // earliest valid candidate of each pair in the chunk
      for (slot = (int)(hash_start(key, kChunkSlots));; slot = (slot + 1) & (kChunkSlots - 1)) {
        const unsigned long long prev = atomicCAS(&ckey[slot], kEmpty, (unsigned long long)key);
        if (prev == kEmpty || prev == key) break;
      }
      atomicMin(&cmin[slot], (int)threadIdx.x);
    }
    __syncthreads();
    const bool first = valid && cmin[slot] == (int)threadIdx.x;
    int t;
    const int r = block_scan_flag<kWarps>(first, sh, t);   // its barriers order every cmin read before the reset below
    if (valid) ckey[slot] = kEmpty, cmin[slot] = kThreads;
    if (first && taken + r < quota) {
      const int64_t at = o + taken + r;
      if (at < capacity) staged[at] = ((unsigned long long)b << 32) | a;
      F.add(a, b);
    }
    taken += (int64_t)t < quota - taken ? (int64_t)t : quota - taken;
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[g] = taken;
}

__global__ void __launch_bounds__(32)
k_negative_count_scan(const int64_t* __restrict__ counts, int64_t B, int64_t* __restrict__ off) {
  pdl_prologue();
  warp_scan_to(B, off, [&](int64_t i) { return counts[i]; });
}

// row 0 at out[off[g] + r], row 1 at out[M + off[g] + r]: the contiguous [2, M] of torch.cat(..., dim=-1)
__global__ void __launch_bounds__(kThreads)
k_negative_fill(const int64_t* __restrict__ node_off, const int64_t* __restrict__ cap_off, const int64_t* __restrict__ off, int64_t B,
                int64_t capacity, const unsigned long long* __restrict__ staged, int64_t* __restrict__ out) {
  pdl_prologue();
  const int64_t g = blockIdx.x, M = off[B], o = off[g], cnt = off[g + 1] - o, s = cap_off[g], n0 = node_off[g];
  for (int64_t r = threadIdx.x; r < cnt && s + r < capacity; r += kThreads) {
    const unsigned long long p = staged[s + r];
    out[o + r] = n0 + (int64_t)(p & 0xffffffffull);
    out[M + o + r] = n0 + (int64_t)(p >> 32);
  }
}

struct Layout {
  int64_t cap_off, counts, staged, hash, total;
};
Layout layout(int64_t B, int64_t E, int64_t capacity) {
  Layout L;
  L.cap_off = 0;
  L.counts = L.cap_off + align_up((B + 1) * 8, 256);
  L.staged = L.counts + align_up((B > 0 ? B : 1) * 8, 256);
  L.hash = L.staged + align_up((capacity > 0 ? capacity : 1) * 8, 256);
  L.total = L.hash + align_up((E > 0 ? E : 1) * kHashPerColumn * 8, 256);
  return L;
}

}  // namespace

extern "C" {

int64_t pgnn_negative_edges_capacity(const int64_t* edge_off_host, int64_t B) {
  if (!edge_off_host || B < 0) return PGNN_EINVAL;
  int64_t c = 0;
  for (int64_t g = 0; g < B; ++g) c += neg_capacity(edge_off_host[g + 1] - edge_off_host[g]);
  return c;
}

int64_t pgnn_negative_edges_workspace_bytes(int64_t B, int64_t E, int64_t capacity) {
  if (B < 0 || E < 0 || capacity < 0) return PGNN_EINVAL;
  return layout(B, E, capacity).total;
}

int pgnn_negative_edges(const int64_t* edge_index, int64_t E, const int64_t* node_off, const int64_t* edge_off, int64_t B, int64_t seed,
                        int64_t capacity, void* workspace, int64_t workspace_bytes, int64_t* negative_edge_index,
                        int64_t* negative_edge_off, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && E >= 0 && capacity >= 0 && node_off && edge_off && negative_edge_off && workspace);
  PGNN_CHECK_ARG(E == 0 || edge_index);
  PGNN_CHECK_ARG(capacity == 0 || negative_edge_index);
  if (workspace_bytes < pgnn_negative_edges_workspace_bytes(B, E, capacity)) return PGNN_EWORKSPACE;
  const Layout L = layout(B, E, capacity);
  char* w = reinterpret_cast<char*>(workspace);
  int64_t* cap_off = reinterpret_cast<int64_t*>(w + L.cap_off);
  int64_t* counts = reinterpret_cast<int64_t*>(w + L.counts);
  unsigned long long* staged = reinterpret_cast<unsigned long long*>(w + L.staged);
  unsigned long long* hash = reinterpret_cast<unsigned long long*>(w + L.hash);
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(pgnn_launch(k_negative_capacity_scan, dim3(1), dim3(32), 0, st, edge_off, B, cap_off));
  PGNN_LAUNCH_CHECK();
  if (B > 0) {
    PGNN_CUDA(cudaFuncSetAttribute(k_negative_select, cudaFuncAttributeMaxDynamicSharedMemorySize, kBitmapBytes));
    PGNN_CUDA(pgnn_launch(k_negative_select, dim3((unsigned)B), dim3(kThreads), (size_t)kBitmapBytes, st, edge_index, E, node_off, edge_off,
                          (uint64_t)seed, (const int64_t*)cap_off, capacity, hash, staged, counts, pgnn_error_flag_ptr()));
    PGNN_LAUNCH_CHECK();
  }
  PGNN_CUDA(pgnn_launch(k_negative_count_scan, dim3(1), dim3(32), 0, st, (const int64_t*)counts, B, negative_edge_off));
  PGNN_LAUNCH_CHECK();
  if (B > 0) {
    PGNN_CUDA(pgnn_launch(k_negative_fill, dim3((unsigned)B), dim3(kThreads), 0, st, node_off, (const int64_t*)cap_off,
                          (const int64_t*)negative_edge_off, B, capacity, (const unsigned long long*)staged, negative_edge_index));
    PGNN_LAUNCH_CHECK();
  }
  return PGNN_OK;
}

}  // extern "C"
