// ExtractSubstructureContextPair on the device (SURVEY.md section 8(f), row f4): chem/util.py:55-151 (through the networkx
// round trip of chem/loader.py:146-221) and bio/util.py:123-205, fused with BatchSubstructContext.from_data_list
// (chem/batch.py:141-210, bio/batch.py:196-265).  The reference runs a networkx BFS and three Python loops per sample on
// DataLoader workers; here the dataset stays in HBM (data.MoleculeStore / BioGraphStore) and a batch of (substructure,
// context) pairs is three launches over the selected graphs:
//
//   k_extract_bfs     one CTA per graph: hop distance from the root by level-synchronous sweeps over the graph's bond
//                     pairs (the undirected graph of the even-indexed edge_index columns, chem/loader.py:169; a pair whose
//                     endpoints already occurred is skipped, :173 -> the store's `pair_first` bits), membership
//                     substructure = ball(k), context = ball(l1) xor ball(l2) (bio: everything / outside ball(l1)),
//                     new node numbers (ascending original index) and the five sizes of the pair
//   k_extract_scan    exclusive scans of the sizes over the batch; a pair without context is dropped (chem/batch.py:168)
//   k_extract_fill_*  relabelled node features, both directions of every kept bond adjacent ((i,j),(j,i), same attribute
//                     row: nx_to_graph_data_obj_simple, chem/loader.py:201-207), centre, overlap list with its segment
//                     ids and sizes, each offset by the running node count of its side
//
// Ordering is defined by oracle/step_io_oracle.py (header there: the reference's own numbering is networkx / CPython set
// iteration order, which no consumer depends on); against that restatement everything here is integer work and bit-exact.
// The output sizes are data dependent: the caller allocates at the upper bounds it knows on the host (the full graphs'
// node and edge counts) and reads the six totals back (48 bytes) to narrow its views; edge_index is written compactly
// ([2, total] with the total taken from the scan on the device), so the narrowed views are contiguous.
#include "common.cuh"

namespace {

constexpr int kInf = 1 << 30;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
enum { Q_NS = 0, Q_ES, Q_NC, Q_EC, Q_KO, Q_KEPT, Q_COUNT };

struct Ws {
  int64_t *full_node_off, *counts;  // [B+1], [Q_COUNT][B]
  int32_t *root, *dist, *map_s, *map_c;  // [B], [Nfull] x 3
  int64_t total;
};

__host__ Ws carve(void* base, int64_t B, int64_t nfull) {
  Ws w;
  char* p = reinterpret_cast<char*>(base);
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    char* q = p + off;
    off += align_up(bytes > 0 ? bytes : 1, 256);
    return q;
  };
  w.full_node_off = reinterpret_cast<int64_t*>(take((B + 1) * 8));
  w.counts = reinterpret_cast<int64_t*>(take(Q_COUNT * B * 8));
  w.root = reinterpret_cast<int32_t*>(take(B * 4));
  w.dist = reinterpret_cast<int32_t*>(take(nfull * 4));
  w.map_s = reinterpret_cast<int32_t*>(take(nfull * 4));
  w.map_c = reinterpret_cast<int32_t*>(take(nfull * 4));
  w.total = off;
  return w;
}

// exclusive prefix of two flags across the CTA (ascending thread index); returns the CTA totals in ta / tb
__device__ __forceinline__ void block_scan2(bool a, bool b, int (*sh)[kWarps], int& pa, int& pb, int& ta, int& tb) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ma = __ballot_sync(0xffffffffu, a), mb = __ballot_sync(0xffffffffu, b);
  const unsigned lt = (1u << lane) - 1u;
  __syncthreads();  // previous use of sh is over
  if (lane == 0) {
    sh[0][warp] = __popc(ma);
    sh[1][warp] = __popc(mb);
  }
  __syncthreads();
  pa = __popc(ma & lt);
  pb = __popc(mb & lt);
  ta = tb = 0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    const int ca = sh[0][w], cb = sh[1][w];
    if (w < warp) {
      pa += ca;
      pb += cb;
    }
    ta += ca;
    tb += cb;
  }
}

// node offsets of the FULL selected graphs (the workspace's dist / map arrays are laid out by them): one warp, any B
__global__ void __launch_bounds__(32)
k_extract_full_off(const int64_t* __restrict__ node_ptr, const int64_t* __restrict__ ids, int64_t B, int64_t* __restrict__ off) {
  pdl_prologue();
  const int lane = threadIdx.x;
  int64_t carry = 0;
  for (int64_t base = 0; base < B; base += 32) {
    const int64_t i = base + lane;
    int64_t n = 0;
    if (i < B) n = node_ptr[ids[i] + 1] - node_ptr[ids[i]];
    int64_t s = n;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (i < B) off[i] = carry + s - n;
    carry += __shfl_sync(0xffffffffu, s, 31);
  }
  if (lane == 0) off[B] = carry;
}

__device__ __forceinline__ bool in_ball(int d, int cutoff) { return d <= (cutoff > 0 ? cutoff : 0); }  // chem/util.py:73-78: 0 -> -1 -> {root}

__global__ void __launch_bounds__(kThreads)
k_extract_bfs(const int64_t* __restrict__ node_ptr, const int64_t* __restrict__ edge_ptr, const int32_t* __restrict__ sei, int64_t store_edges,
              const uint8_t* __restrict__ pair_first, const int64_t* __restrict__ ids, int64_t B, const int32_t* __restrict__ roots, uint64_t seed,
              int k, int l1, int l2, int whole, const int64_t* __restrict__ full_off, int32_t* __restrict__ root_out, int32_t* __restrict__ dist_all,
              int32_t* __restrict__ map_s_all, int32_t* __restrict__ map_c_all, int64_t* __restrict__ counts, unsigned int* __restrict__ err) {
  pdl_prologue();
  __shared__ int sh[2][kWarps];
  __shared__ int changed, cnt_es, cnt_ec;
  const int64_t i = blockIdx.x;
  const int64_t g = ids[i];
  const int n = (int)(node_ptr[g + 1] - node_ptr[g]);
  const int64_t e0 = edge_ptr[g];
  const int m = (int)((edge_ptr[g + 1] - e0) >> 1);
  const int64_t no = full_off[i];
  int32_t* dist = dist_all + no;
  int32_t* map_s = map_s_all + no;
  int32_t* map_c = map_c_all + no;
  const int32_t* src = sei + e0;
  const int32_t* dst = sei + store_edges + e0;
  const uint8_t* first = pair_first + (e0 >> 1);
  int root = 0;
  if (n > 0) {
    if (roots) {
      root = roots[i];
      if (root < 0 || root >= n) {
        if (threadIdx.x == 0 && err) atomicOr(err, PGNN_DEVERR_NODE_ID);
        root = root < 0 ? 0 : n - 1;
      }
    } else {
      root = (int)(splitmix64(seed, (uint64_t)i) % (uint64_t)n);
    }
  }
  for (int v = threadIdx.x; v < n; v += kThreads) dist[v] = v == root ? 0 : kInf;
  if (threadIdx.x == 0) {
    root_out[i] = root;
    cnt_es = cnt_ec = 0;
  }
  const int c_k = k > 0 ? k : 0, c_1 = l1 > 0 ? l1 : 0, c_2 = l2 > 0 ? l2 : 0;
  const int maxd = whole ? c_1 : (c_k > c_1 ? (c_k > c_2 ? c_k : c_2) : (c_1 > c_2 ? c_1 : c_2));
  __syncthreads();
  for (int level = 1; level <= maxd; ++level) {
    if (threadIdx.x == 0) changed = 0;
    __syncthreads();
    for (int p = threadIdx.x; p < m; p += kThreads) {
      if (!first[p]) continue;
      const int u = src[2 * p], v = dst[2 * p];
      if ((unsigned)u >= (unsigned)n || (unsigned)v >= (unsigned)n) {
        if (err) atomicOr(err, PGNN_DEVERR_NODE_ID);
        continue;
      }
      const int du = dist[u], dv = dist[v];
      if (du == level - 1 && dv == kInf) {
        dist[v] = level;
        changed = 1;
      } else if (dv == level - 1 && du == kInf) {
        dist[u] = level;
        changed = 1;
      }
    }
    __syncthreads();
    const int c = changed;
    __syncthreads();
    if (!c) break;
  }
  // membership and new numbering (ascending original index)
  int carry_s = 0, carry_c = 0, overlap = 0;
  for (int base = 0; base < n; base += kThreads) {
    const int v = base + threadIdx.x;
    bool a = false, b = false;
    if (v < n) {
      const int d = dist[v];
      a = whole ? true : in_ball(d, k);
      b = whole ? !in_ball(d, l1) : (in_ball(d, l1) != in_ball(d, l2));
    }
    int pa, pb, ta, tb;
    block_scan2(a, b, sh, pa, pb, ta, tb);
    if (v < n) {
      map_s[v] = a ? carry_s + pa : -1;
      map_c[v] = b ? carry_c + pb : -1;
    }
    int po, pd, to, td;
    block_scan2(a && b, false, sh, po, pd, to, td);
    carry_s += ta;
    carry_c += tb;
    overlap += to;
  }
  __syncthreads();
  int es = 0, ec = 0;
  for (int p = threadIdx.x; p < m; p += kThreads) {
    if (!first[p]) continue;
    const int u = src[2 * p], v = dst[2 * p];
    if ((unsigned)u >= (unsigned)n || (unsigned)v >= (unsigned)n) continue;
    es += (map_s[u] >= 0 && map_s[v] >= 0);
    ec += (map_c[u] >= 0 && map_c[v] >= 0);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    es += __shfl_xor_sync(0xffffffffu, es, o);
    ec += __shfl_xor_sync(0xffffffffu, ec, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&cnt_es, es);
    atomicAdd(&cnt_ec, ec);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const bool keep = carry_c > 0;  // chem/batch.py:168: "If there is no context, just skip!!"
    counts[Q_NS * B + i] = keep ? carry_s : 0;
    counts[Q_ES * B + i] = keep ? 2 * cnt_es : 0;
    counts[Q_NC * B + i] = keep ? carry_c : 0;
    counts[Q_EC * B + i] = keep ? 2 * cnt_ec : 0;
    counts[Q_KO * B + i] = keep ? overlap : 0;
    counts[Q_KEPT * B + i] = keep ? 1 : 0;
  }
}

// warp q: offsets[q][0..B] = exclusive scan of counts[q][0..B)
__global__ void __launch_bounds__(32 * Q_COUNT)
k_extract_scan(const int64_t* __restrict__ counts, int64_t B, int64_t* __restrict__ offsets) {
  pdl_prologue();
  const int lane = threadIdx.x & 31, q = threadIdx.x >> 5;
  const int64_t* c = counts + (int64_t)q * B;
  int64_t* o = offsets + (int64_t)q * (B + 1);
  int64_t carry = 0;
  for (int64_t base = 0; base < B; base += 32) {
    const int64_t i = base + lane;
    const int64_t n = i < B ? c[i] : 0;
    int64_t s = n;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (i < B) o[i] = carry + s - n;
    carry += __shfl_sync(0xffffffffu, s, 31);
  }
  if (lane == 0) o[B] = carry;
}

struct Side {            // one side (substructure or context) of the batch being written
  int64_t node_off, edge_off, edge_total;
  const int32_t* map;
};

// both directions of every kept bond pair, adjacent, in source order (chem/loader.py:201-207)
template <typename WriteAttr>
__device__ __forceinline__ void fill_edges(const Side& a, const Side& b, int m, int n, const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                           const uint8_t* __restrict__ first, int (*sh)[kWarps], int64_t* __restrict__ ei_a, int64_t* __restrict__ ei_b,
                                           WriteAttr write_attr) {
  int carry_a = 0, carry_b = 0;
  for (int base = 0; base < m; base += kThreads) {
    const int p = base + threadIdx.x;
    bool fa = false, fb = false;
    int u = 0, v = 0;
    if (p < m && first[p]) {
      u = src[2 * p];
      v = dst[2 * p];
      if ((unsigned)u < (unsigned)n && (unsigned)v < (unsigned)n) {
        fa = a.map && a.map[u] >= 0 && a.map[v] >= 0;
        fb = b.map[u] >= 0 && b.map[v] >= 0;
      }
    }
    int pa, pb, ta, tb;
    block_scan2(fa, fb, sh, pa, pb, ta, tb);
    if (fa) {
      const int64_t col = a.edge_off + 2 * (int64_t)(carry_a + pa);
      const int64_t nu = a.node_off + a.map[u], nv = a.node_off + a.map[v];
      ei_a[col] = nu;
      ei_a[a.edge_total + col] = nv;
      ei_a[col + 1] = nv;
      ei_a[a.edge_total + col + 1] = nu;
      write_attr(0, col, p);
    }
    if (fb) {
      const int64_t col = b.edge_off + 2 * (int64_t)(carry_b + pb);
      const int64_t nu = b.node_off + b.map[u], nv = b.node_off + b.map[v];
      ei_b[col] = nu;
      ei_b[b.edge_total + col] = nv;
      ei_b[col + 1] = nv;
      ei_b[b.edge_total + col + 1] = nu;
      write_attr(1, col, p);
    }
    carry_a += ta;
    carry_b += tb;
  }
}

__device__ __forceinline__ void fill_overlap(int n, const int32_t* __restrict__ map_s, const int32_t* __restrict__ map_c, int64_t nc_off, int64_t ko_off,
                                             int64_t ordinal, int (*sh)[kWarps], int64_t* __restrict__ overlap, int64_t* __restrict__ seg) {
  int carry = 0;
  for (int base = 0; base < n; base += kThreads) {
    const int v = base + threadIdx.x;
    const bool f = v < n && (map_s ? map_s[v] >= 0 : true) && map_c[v] >= 0;
    int pa, pb, ta, tb;
    block_scan2(f, false, sh, pa, pb, ta, tb);
    if (f) {
      overlap[ko_off + carry + pa] = nc_off + map_c[v];
      seg[ko_off + carry + pa] = ordinal;
    }
    carry += ta;
  }
}

__global__ void __launch_bounds__(kThreads)
k_extract_fill_chem(const int64_t* __restrict__ node_ptr, const int64_t* __restrict__ edge_ptr, const uint8_t* __restrict__ sx,
                    const int32_t* __restrict__ sei, int64_t store_edges, const uint8_t* __restrict__ sea, const uint8_t* __restrict__ pair_first,
                    const int64_t* __restrict__ ids, int64_t B, const int64_t* __restrict__ full_off, const int32_t* __restrict__ root_all,
                    const int32_t* __restrict__ map_s_all, const int32_t* __restrict__ map_c_all, const int64_t* __restrict__ counts,
                    const int64_t* __restrict__ off, int64_t* __restrict__ x_s, int64_t* __restrict__ ei_s, int64_t* __restrict__ ea_s,
                    int64_t* __restrict__ center, int64_t* __restrict__ x_c, int64_t* __restrict__ ei_c, int64_t* __restrict__ ea_c,
                    int64_t* __restrict__ overlap, int64_t* __restrict__ seg, int64_t* __restrict__ sizes) {
  pdl_prologue();
  __shared__ int sh[2][kWarps];
  const int64_t i = blockIdx.x;
  if (!counts[Q_KEPT * B + i]) return;
  const int64_t g = ids[i], B1 = B + 1;
  const int n = (int)(node_ptr[g + 1] - node_ptr[g]);
  const int64_t n0 = node_ptr[g], e0 = edge_ptr[g];
  const int m = (int)((edge_ptr[g + 1] - e0) >> 1);
  const int32_t* map_s = map_s_all + full_off[i];
  const int32_t* map_c = map_c_all + full_off[i];
  const Side S{off[Q_NS * B1 + i], off[Q_ES * B1 + i], off[Q_ES * B1 + B], map_s};
  const Side C{off[Q_NC * B1 + i], off[Q_EC * B1 + i], off[Q_EC * B1 + B], map_c};
  const int64_t ordinal = off[Q_KEPT * B1 + i], ko_off = off[Q_KO * B1 + i];
  for (int v = threadIdx.x; v < n; v += kThreads) {
    const int64_t a = sx[2 * (n0 + v)], b = sx[2 * (n0 + v) + 1];
    if (map_s[v] >= 0) {
      x_s[2 * (S.node_off + map_s[v])] = a;
      x_s[2 * (S.node_off + map_s[v]) + 1] = b;
    }
    if (map_c[v] >= 0) {
      x_c[2 * (C.node_off + map_c[v])] = a;
      x_c[2 * (C.node_off + map_c[v]) + 1] = b;
    }
  }
  if (threadIdx.x == 0) {
    center[ordinal] = S.node_off + map_s[root_all[i]];      // chem/util.py:119-121 + the batch offset (chem/batch.py:185-188)
    sizes[ordinal] = counts[Q_KO * B + i];
  }
  fill_overlap(n, map_s, map_c, C.node_off, ko_off, ordinal, sh, overlap, seg);
  const uint8_t* ea = sea + 2 * e0;
  fill_edges(S, C, m, n, sei + e0, sei + store_edges + e0, pair_first + (e0 >> 1), sh, ei_s, ei_c, [&](int side, int64_t col, int p) {
    int64_t* o = side ? ea_c : ea_s;
    const int64_t t = ea[4 * p], d = ea[4 * p + 1];   // attribute row of the pair's first column (edge 2p)
    o[2 * col] = t;
    o[2 * col + 1] = d;
    o[2 * col + 2] = t;
    o[2 * col + 3] = d;
  });
}

// bio: the substructure is the whole ego graph (bio/util.py:170-174: the caller's ordinary collation), only the context side
// and the overlap list (every context node, :195-203) are produced.  nx_to_graph_data_obj (bio/loader.py:76-116) re-emits the
// seven w bits and zeros for the self-loop / mask columns.
__global__ void __launch_bounds__(kThreads)
k_extract_fill_bio(const int64_t* __restrict__ node_ptr, const int64_t* __restrict__ edge_ptr, const int32_t* __restrict__ sei, int64_t store_edges,
                   const uint16_t* __restrict__ sbits, const uint8_t* __restrict__ pair_first, const int64_t* __restrict__ ids, int64_t B,
                   const int64_t* __restrict__ full_off, const int32_t* __restrict__ map_c_all, const int64_t* __restrict__ counts,
                   const int64_t* __restrict__ off, float* __restrict__ x_c, int64_t* __restrict__ ei_c, float* __restrict__ ea_c,
                   int64_t* __restrict__ overlap, int64_t* __restrict__ seg, int64_t* __restrict__ sizes) {
  pdl_prologue();
  __shared__ int sh[2][kWarps];
  const int64_t i = blockIdx.x;
  if (!counts[Q_KEPT * B + i]) return;
  const int64_t g = ids[i], B1 = B + 1;
  const int n = (int)(node_ptr[g + 1] - node_ptr[g]);
  const int64_t e0 = edge_ptr[g];
  const int m = (int)((edge_ptr[g + 1] - e0) >> 1);
  const int32_t* map_c = map_c_all + full_off[i];
  const Side S{0, 0, 0, nullptr};
  const Side C{off[Q_NC * B1 + i], off[Q_EC * B1 + i], off[Q_EC * B1 + B], map_c};
  const int64_t ordinal = off[Q_KEPT * B1 + i], ko_off = off[Q_KO * B1 + i];
  for (int v = threadIdx.x; v < n; v += kThreads)
    if (map_c[v] >= 0) x_c[C.node_off + map_c[v]] = 1.f;
  if (threadIdx.x == 0) sizes[ordinal] = counts[Q_KO * B + i];
  fill_overlap(n, nullptr, map_c, C.node_off, ko_off, ordinal, sh, overlap, seg);
  const uint16_t* bits = sbits + e0;
  fill_edges(S, C, m, n, sei + e0, sei + store_edges + e0, pair_first + (e0 >> 1), sh, (int64_t*)nullptr, ei_c, [&](int side, int64_t col, int p) {
    const unsigned w = bits[2 * p] & 0x7Fu;
#pragma unroll
    for (int q = 0; q < 9; ++q) {
      const float f = (w >> q) & 1u ? 1.f : 0.f;
      ea_c[col * 9 + q] = f;
      ea_c[(col + 1) * 9 + q] = f;
    }
  });
}

}  // namespace

extern "C" {

int64_t pgnn_extract_pairs_workspace_bytes(int64_t B, int64_t full_nodes) {
  if (B < 0 || full_nodes < 0) return PGNN_EINVAL;
  return carve(nullptr, B, full_nodes).total;
}

int pgnn_extract_pairs(const int64_t* node_ptr, const int64_t* edge_ptr, const int32_t* store_edge_index, int64_t store_num_edges,
                       const uint8_t* pair_first, const int64_t* graph_ids, int64_t B, int64_t full_nodes, const int32_t* roots, int64_t seed, int k,
                       int l1, int l2, int whole_graph, void* workspace, int64_t workspace_bytes, int64_t* offsets, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && full_nodes >= 0 && store_num_edges >= 0 && node_ptr && edge_ptr && offsets && workspace);
  if (B > 0) PGNN_CHECK_ARG(graph_ids && (store_num_edges == 0 || (store_edge_index && pair_first)));
  const Ws w = carve(workspace, B, full_nodes);
  if (workspace_bytes < w.total) return PGNN_EWORKSPACE;
  cudaStream_t st = as_stream(stream);
  PGNN_CUDA(pgnn_launch(k_extract_full_off, dim3(1), dim3(32), 0, st, node_ptr, graph_ids, B, w.full_node_off));
  PGNN_LAUNCH_CHECK();
  if (B > 0) {
    PGNN_CUDA(pgnn_launch(k_extract_bfs, dim3((unsigned)B), dim3(kThreads), 0, st, node_ptr, edge_ptr, store_edge_index, store_num_edges, pair_first,
                          graph_ids, B, roots, (uint64_t)seed, k, l1, l2, whole_graph, (const int64_t*)w.full_node_off, w.root, w.dist, w.map_s, w.map_c,
                          w.counts, pgnn_error_flag_ptr()));
    PGNN_LAUNCH_CHECK();
  }
  PGNN_CUDA(pgnn_launch(k_extract_scan, dim3(1), dim3(32 * Q_COUNT), 0, st, (const int64_t*)w.counts, B, offsets));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_extract_fill_chem(const int64_t* node_ptr, const int64_t* edge_ptr, const uint8_t* store_x, const int32_t* store_edge_index,
                           int64_t store_num_edges, const uint8_t* store_edge_attr, const uint8_t* pair_first, const int64_t* graph_ids, int64_t B,
                           int64_t full_nodes, const void* workspace, const int64_t* offsets, int64_t* x_substruct, int64_t* edge_index_substruct,
                           int64_t* edge_attr_substruct, int64_t* center_substruct_idx, int64_t* x_context, int64_t* edge_index_context,
                           int64_t* edge_attr_context, int64_t* overlap_context_substruct_idx, int64_t* batch_overlapped_context,
                           int64_t* overlapped_context_size, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && full_nodes >= 0 && workspace && offsets);
  if (B == 0) return PGNN_OK;
  PGNN_CHECK_ARG(node_ptr && edge_ptr && store_x && graph_ids && x_substruct && edge_index_substruct && edge_attr_substruct && center_substruct_idx &&
                 x_context && edge_index_context && edge_attr_context && overlap_context_substruct_idx && batch_overlapped_context &&
                 overlapped_context_size);
  const Ws w = carve(const_cast<void*>(workspace), B, full_nodes);
  PGNN_CUDA(pgnn_launch(k_extract_fill_chem, dim3((unsigned)B), dim3(kThreads), 0, as_stream(stream), node_ptr, edge_ptr, store_x, store_edge_index,
                        store_num_edges, store_edge_attr, pair_first, graph_ids, B, (const int64_t*)w.full_node_off, (const int32_t*)w.root,
                        (const int32_t*)w.map_s, (const int32_t*)w.map_c, (const int64_t*)w.counts, offsets, x_substruct, edge_index_substruct,
                        edge_attr_substruct, center_substruct_idx, x_context, edge_index_context, edge_attr_context, overlap_context_substruct_idx,
                        batch_overlapped_context, overlapped_context_size));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

int pgnn_extract_fill_bio(const int64_t* node_ptr, const int64_t* edge_ptr, const int32_t* store_edge_index, int64_t store_num_edges,
                          const uint16_t* store_edge_bits, const uint8_t* pair_first, const int64_t* graph_ids, int64_t B, int64_t full_nodes,
                          const void* workspace, const int64_t* offsets, float* x_context, int64_t* edge_index_context, float* edge_attr_context,
                          int64_t* overlap_context_substruct_idx, int64_t* batch_overlapped_context, int64_t* overlapped_context_size, void* stream) {
  PGNN_CHECK_ARG(B >= 0 && full_nodes >= 0 && workspace && offsets);
  if (B == 0) return PGNN_OK;
  PGNN_CHECK_ARG(node_ptr && edge_ptr && graph_ids && x_context && edge_index_context && edge_attr_context && overlap_context_substruct_idx &&
                 batch_overlapped_context && overlapped_context_size);
  const Ws w = carve(const_cast<void*>(workspace), B, full_nodes);
  PGNN_CUDA(pgnn_launch(k_extract_fill_bio, dim3((unsigned)B), dim3(kThreads), 0, as_stream(stream), node_ptr, edge_ptr, store_edge_index,
                        store_num_edges, store_edge_bits, pair_first, graph_ids, B, (const int64_t*)w.full_node_off, (const int32_t*)w.map_c,
                        (const int64_t*)w.counts, offsets, x_context, edge_index_context, edge_attr_context, overlap_context_substruct_idx,
                        batch_overlapped_context, overlapped_context_size));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

}  // extern "C"
