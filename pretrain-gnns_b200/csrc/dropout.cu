// Dropout as an operator (chem/model.py:271-275, bio/model.py:283-286: F.dropout(h, drop_ratio, training)) for the
// layer-by-layer composition.  The mask is the library's counter-hash draw (PgnnDropout, common.cuh): the backward regenerates it
// from (seed, layer) instead of reading a stored mask.  The whole-encoder path applies the same mask inside its BatchNorm and
// gather kernels (norm.cu, aggregate.cu).
#include "common.cuh"

namespace {

// one thread per (row, column); the grid-stride loop keeps the hash cost off the memory pipe's critical path
__global__ void __launch_bounds__(256)
k_dropout(const float* __restrict__ x, int64_t ldx, int64_t M, int64_t C, PgnnDropout d, float* __restrict__ y, int64_t ldy) {
  pdl_prologue();
  const int64_t total = M * C;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / C;
    const int64_t c = idx - r * C;
    y[r * ldy + c] = x[r * ldx + c] * dropout_factor(d, r, C, c);
  }
}

// forward and backward are the same map: y = x * factor(l, i, c)
int dropout_apply(const float* x, int64_t ldx, int64_t M, int64_t C, float p, int64_t seed, int64_t layer, float* y, int64_t ldy,
                  void* stream) {
  PgnnDropout d;
  PGNN_CHECK_ARG(M >= 0 && C > 0 && layer >= 0 && layer < (1ll << 24) && pgnn_make_dropout(p, seed, layer, &d));
  PGNN_CHECK_ARG(M * C < (1ll << 40));  // the element index must stay below the layer bits
  if (M == 0) return PGNN_OK;
  PGNN_CHECK_ARG(x && y && ldx >= C && ldy >= C);
  PGNN_CUDA(pgnn_launch(k_dropout, dim3(grid_items(M * C, 256)), dim3(256), 0, as_stream(stream), x, ldx, M, C, d, y, ldy));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

}  // namespace

extern "C" {

int pgnn_dropout_fwd(const float* x, int64_t ldx, int64_t M, int64_t C, float p, int64_t seed, int64_t layer, float* y, int64_t ldy,
                     void* stream) {
  return dropout_apply(x, ldx, M, C, p, seed, layer, y, ldy, stream);
}

int pgnn_dropout_bwd(const float* gy, int64_t ldgy, int64_t M, int64_t C, float p, int64_t seed, int64_t layer, float* gx,
                     int64_t ldgx, void* stream) {
  return dropout_apply(gy, ldgy, M, C, p, seed, layer, gx, ldgx, stream);
}

}  // extern "C"
