// Dense node transforms on the Hopper tensor cores (precision 1): error-compensated 3xTF32 with wgmma.
//
// fp32 parity (1e-4, north_star) rules out plain TF32 (10-bit mantissa over K = 300/600).  Every fp32 operand x
// is split into hi = trunc_tf32(x) and lo = x - hi (exact in fp32); each k-step issues three wgmma (lo*hi, hi*lo,
// hi*hi).  The dropped lo*lo term and the truncation of lo are ~2^-20 relative: the GEMM error is of the same class
// as an fp32 FFMA GEMM (tools/check_tc.py).
//
// One kernel template serves the three operand layouts of dense.cu (same roles, same epilogues):
//   fwd    y[M,N]  = x[M,K]  . w[N,K]^T      A K-major,  B K-major
//   dgrad  gx[M,K] = gy[M,N] . w[N,K]        A K-major,  B MN-major (w rows are the reduction)
//   wgrad  gw[N,K] = gy[M,N]^T . x[M,K]      A MN-major, B MN-major (node rows are the reduction; split-K)
//
// Structure (per CTA: one 128 x BN output tile, two warpgroups of 64 rows each, BK = 32 per block):
//   * A comes from registers (the RS form of wgmma): each thread holds its rows of the tf32 A fragment and splits them
//     into hi / lo in registers.  Block kb + 1 of A is copied raw into the other of two shared-memory buffers with
//     cp.async while block kb runs (no registers held by the copy), and read from there into the fragment.  Within a block
//     the reduction index is permuted (kperm) so that a thread's fragment slots are two 16-byte pieces of each of its
//     rows: one 16-byte shared-memory read per row and two k-steps for a K-major A; an MN-major A (wgrad's gy^T) is read
//     element by element.
//   * B goes through NSTAGE shared-memory stages: every thread loads its share of block kb + 1 (16-byte global loads
//     along whichever extent is contiguous, zero-filled out of range) while the tensor cores work on block kb, then
//     splits it into hi / lo and stores both, permuted like A, in the K-major 128B-swizzled layout (tf32 wgmma reads a
//     K-major B only, so an MN-major source is transposed on this store), and fences the stores to the async proxy;
//   * B_IMG (K-major A and B only): B is a weight, the same for the whole pass, so it is split and laid out once per pass into a
//     pre-split image (see kperm below) and every stage is filled by cp.async 16-byte copies, two blocks ahead, in the commit
//     group of an A copy: no registers, no split and no scalar stores in the mainloop, and no global load in front of a barrier;
//   * per k-step and warpgroup: one commit group of 3 wgmma.m64nBNk8 (lo*hi, hi*lo into the cross-term accumulator,
//     hi*hi into its own), A fragments in FRAG_SETS register sets.  A set is rewritten only after wait_group has
//     retired the group that read it, so FRAG_SETS - 1 groups stay queued across k-steps, k-blocks and the one barrier
//     per block; with three B stages that barrier is also what frees the stage the next block is stored into;
//   * epilogue: both accumulators are summed into a shared-memory staging tile, then written out row-contiguously
//     with bias / ReLU / mask applied, plus the optional fused column reductions.
#include <cstdlib>

#include "common.cuh"

namespace {

constexpr int BM = 128;        // rows per CTA: two warpgroups x wgmma M = 64
constexpr int BK = 32;         // fp32 of the reduction per block = one 128-byte swizzle row
constexpr int NTHREADS = 256;  // two warpgroups; every thread loads, converts, issues its warpgroup's wgmma and runs the epilogue

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// byte offset of element (r, k) in a K-major SWIZZLE_128B tile: 8-row groups of 1024 B, the 16-byte chunk index XOR-ed
// with the row index mod 8
__device__ __forceinline__ int sw128_off(int r, int k) { return (r >> 3) * 1024 + (r & 7) * 128 + ((((k >> 2) ^ (r & 7))) << 4) + (k & 3) * 4; }

// wgmma shared-memory matrix descriptor (sm_90): start >> 4 | LBO >> 4 << 16 (unused for swizzled K-major) | SBO >> 4 << 32 |
// layout 1 (128B swizzle) << 62
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N of this warpgroup's commit groups still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// d[64 x 64] += a[64 x 8] . b[64 x 8]^T: tf32 A fragment from registers, B from shared memory, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_tf32_m64n64k8_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db)
      : "memory");
}
// d[64 x 128] += a[64 x 8] . b[128 x 8]^T, as above
__device__ __forceinline__ void wgmma_tf32_m64n128k8_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db)
      : "memory");
}
template <int BN>
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (BN == 128) wgmma_tf32_m64n128k8_rs(d, a, db);
  else wgmma_tf32_m64n64k8_rs(d, a, db);
}
// keeps the compiler from moving accumulator registers across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// The reduction index k of a block and its slot in the A fragment and the stored B tile: the two base-4 digits of k mod 16
// swap (an involution, so it also maps a slot back to its k).  k-step j, fragment column c (thread t = c mod 4 of its quad)
// then holds k = 16 (j / 2) + 4 t + 2 (j % 2) + c / 4: thread t's slots are k = 4t .. 4t + 3 and 16 + 4t .. 16 + 4t + 3.
__device__ __forceinline__ int kperm(int k) { return (k & 16) | ((k & 3) << 2) | ((k >> 2) & 3); }

// Weight image: a K-major B operand [rows][K] (the GEMM's N extent x its reduction) split once into two planes, hi then lo, each
// [align_up(rows, 128)][align_up(K, 32)] floats, row-major.  Inside every 32-wide block of a row, slot kperm(k) holds element k
// (split_tf32, as the mainloop would split it); padded rows and reduction columns are zero.  So the aligned 16-byte piece at
// (r, 32 kb + 4 c) of a plane is the chunk sw128_off(r mod BN, 4 c) of block kb's stage of that plane: one cp.async16, no tail
// handling, and the zeros are the ones ldg4_tail would have filled in.
constexpr int kImgRows = 128;  // row padding: a whole BN = 64 or 128 tile is always inside the image
__host__ __device__ constexpr int64_t img_rows(int64_t rows) { return (rows + kImgRows - 1) / kImgRows * kImgRows; }
__host__ __device__ constexpr int64_t img_ld(int64_t k) { return (k + BK - 1) / BK * BK; }

// float offset of element (m, k) of a raw MN-major A block [BK][BM].  The XOR keeps 4-row pieces contiguous and spreads both
// the loader's 16-byte stores (k and k + 1) and the fragment reads (8 rows x 4 threads of a quad) over all 32 banks.
__device__ __forceinline__ int araw_off(int m, int k) { return k * BM + (m ^ ((((k >> 2) & 3) << 3) ^ ((k & 1) << 4))); }

// float offset of element (m, k) of a raw K-major A block [BM][BK]: 16-byte pieces stay whole, and the piece index is XOR-ed with
// 4 (m & 1), so the fragment's 16-byte reads (rows m, m + 1 x the 4 threads of a quad per quarter warp) hit 8 distinct pieces
__device__ __forceinline__ int akc_off(int m, int k) { return m * BK + ((((k >> 2) ^ ((m & 1) << 2))) << 2) + (k & 3); }

// 16-byte global -> shared copy that bypasses the registers; the destination bytes from `bytes` on are zero-filled (0: nothing
// is read)
__device__ __forceinline__ void cp_async16(float* dst, const float* src, int bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// x = hi + lo with hi = trunc_tf32(x).  The add of +0 turns a NaN into a NaN with its payload in the high mantissa bits (the GPU's
// canonical NaN), so that a payload only in the 13 truncated bits does not become Inf; finite values pass unchanged.  A non-finite
// x has lo = NaN: see sum_chains.
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = tf32_trunc(__fadd_rn(x, 0.f));
  lo = x - hi;
}

// hi*hi chain + cross terms.  A non-finite operand makes the cross terms NaN (its lo part is NaN, or Inf meets an exact-zero lo),
// while the hi*hi chain holds what the fp32 GEMM gives: every genuine fp32 NaN (a NaN input, Inf - Inf, Inf * 0) reaches that chain
// as a NaN, so a +-Inf there is the fp32 result.
__device__ __forceinline__ float sum_chains(float acc, float accx) { return isinf(acc) ? acc : acc + accx; }

// p[0 .. 3] with the elements from index n on zero (n <= 0: all zero); one 16-byte load when all four are in range
__device__ __forceinline__ float4 ldg4_tail(const float* p, int n) {
  float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
  if (n > 3) x = __ldg(reinterpret_cast<const float4*>(p));
  else if (n > 0) {
    x.x = __ldg(p);
    if (n > 1) x.y = __ldg(p + 1);
    if (n > 2) x.z = __ldg(p + 2);
  }
  return x;
}

__device__ __forceinline__ float f4_at(const float4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

// Operand tile loader.  KC: source contiguous along the reduction (element (r,k) at src[r*ld + k]); otherwise contiguous
// along the row index (element (r,k) at src[k*ld + r]).  R = rows (MN extent) of the tile.  Each thread owns NV 16-byte
// pieces of a [R x BK] block.  MN-major pieces are assigned so that a warp covers 16 rows x 8 k: 64-byte global segments,
// and the transposing scalar stores spread over 16 banks.  The permuted K-major stores (one scalar per element) hit
// 32 distinct banks per warp.
template <bool KC, int R>
struct Loader {
  static constexpr int NV = R * BK / 4 / NTHREADS;
  static_assert(NV >= 1 && R % 16 == 0, "tile rows");
  const float* base;
  int64_t ld, step;  // step: pointer advance per block, in floats
  int r0, rows;
  float4 v[NV];

  __device__ __forceinline__ static void piece(int f, int& rr, int& kk) {
    if (KC) {
      rr = f >> 3;
      kk = (f & 7) * 4;
    } else {
      const int lane = f & 31, w = f >> 5, G = R / 16;
      rr = ((w % G) * 4 + (lane & 3)) * 4;
      kk = (w / G) * 8 + (lane >> 2);
    }
  }
  __device__ __forceinline__ void init(const float* __restrict__ src, int64_t ld_, int r0_, int rows_, int k0) {
    ld = ld_;
    r0 = r0_;
    rows = rows_;
    step = KC ? (int64_t)BK : (int64_t)BK * ld_;
    base = KC ? src + k0 : src + (int64_t)k0 * ld_;
  }
  // krem = reduction elements left from this block's start
  __device__ __forceinline__ void load(int kb, int krem) {
    const float* blk = base + kb * step;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      int rr, kk;
      piece(threadIdx.x + i * NTHREADS, rr, kk);
      const int gr = r0 + rr;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (KC) {
        if (gr < rows) x = ldg4_tail(blk + (int64_t)gr * ld + kk, krem - kk);
      } else if (kk < krem && gr < rows) {
        x = ldg4_tail(blk + (int64_t)kk * ld + gr, rows - gr);
      }
      v[i] = x;
    }
  }
  // B: hi / lo into the K-major swizzled tile, element k at slot kperm(k)
  __device__ __forceinline__ void store(uint8_t* hi, uint8_t* lo) const {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      int rr, kk;
      piece(threadIdx.x + i * NTHREADS, rr, kk);
      if (!KC) asm volatile("" : "+r"(rr), "+r"(kk));  // recompute the 4 NV store offsets per block rather than hold them in registers
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float h, l;
        split_tf32(f4_at(v[i], q), h, l);
        const int o = KC ? sw128_off(rr, kperm(kk + q)) : sw128_off(rr + q, kperm(kk));
        *reinterpret_cast<float*>(hi + o) = h;
        *reinterpret_cast<float*>(lo + o) = l;
      }
    }
  }
};

// A: block kb of this CTA's 128 rows copied raw into a shared-memory buffer (akc_off / araw_off layout) with cp.async, so the
// copy in flight holds no registers.  Same pieces as Loader<KC, BM>; out-of-range elements are zero-filled.  The caller commits.
template <bool KC>
__device__ __forceinline__ void a_copy(float* dst, const float* __restrict__ A, int64_t lda, int m0, int M, int k0, int krem) {
#pragma unroll
  for (int i = 0; i < Loader<KC, BM>::NV; ++i) {
    int rr, kk;
    Loader<KC, BM>::piece(threadIdx.x + i * NTHREADS, rr, kk);
    const int gr = m0 + rr;
    int n = 0;  // elements of the piece in range
    if (KC) n = gr < M ? min(max(krem - kk, 0), 4) : 0;
    else n = kk < krem ? min(max(M - gr, 0), 4) : 0;
    const float* src = n > 0 ? (KC ? A + (int64_t)gr * lda + k0 + kk : A + (int64_t)(k0 + kk) * lda + gr) : A;
    cp_async16(dst + (KC ? akc_off(rr, kk) : araw_off(rr, kk)), src, 4 * n);
  }
}

// B from a weight image: block kb of this CTA's BN rows (both planes, `plane` floats apart) into one stage with cp.async.  Thread
// pieces as Loader<true, BN>: 8 threads cover one 128-byte row of a plane.  The caller commits.
template <int BN>
__device__ __forceinline__ void b_img_copy(uint8_t* hi, uint8_t* lo, const float* __restrict__ img, int64_t ld, int64_t plane, int n0,
                                           int k0) {
#pragma unroll
  for (int i = 0; i < Loader<true, BN>::NV; ++i) {
    const int f = threadIdx.x + i * NTHREADS, rr = f >> 3, kk = (f & 7) * 4;
    const float* src = img + (int64_t)(n0 + rr) * ld + k0 + kk;
    const int o = sw128_off(rr, kk);
    cp_async16(reinterpret_cast<float*>(hi + o), src, 16);
    cp_async16(reinterpret_cast<float*>(lo + o), src + plane, 16);
  }
}

template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

constexpr int NSTAGE = 3;  // raw B stages: block kb + 1 is stored while blocks kb - 1 and kb may still be read

template <int BN, bool B_IMG = false>
struct TileCfg {
  static constexpr int B_BYTES = BN * BK * 4;
  static constexpr int STAGE = 2 * B_BYTES;      // [B hi | B lo]
  static constexpr int A_RAW = BM * BK * 4;      // one raw A block (16 KiB)
  // Copy distance in blocks.  Raw B: block kb + 1 is loaded and stored during block kb (NSTAGE stages), A one block ahead (two
  // buffers).  Image B: two blocks ahead, so a copy has a whole block of MMAs more to land than the barrier in front of it needs;
  // the stages hold blocks kb - 1 (still read by queued wgmma), kb, kb + 1 and kb + 2 (being copied).  A goes two ahead too where
  // its third buffer fits: BN = 128, 4 x 32 KiB + 3 x 16 KiB = 176 KiB (one CTA per SM); at BN = 64, 4 x 16 KiB + 2 x 16 KiB =
  // 96 KiB keeps two CTAs per SM (a third A buffer, 112 KiB + 1 KiB slack each, would not).
  static constexpr int B_STAGES = B_IMG ? 4 : NSTAGE;
  static constexpr int A_DIST = B_IMG && BN == 128 ? 2 : 1;
  static constexpr int A_BUFS = A_DIST + 1;
  static constexpr int SLD = BN + 4;             // epilogue staging row stride (16-byte aligned rows)
  static constexpr int EPI = BM * SLD * 4 + BM * kMaxHookQ * 4;  // staging tile + the hooks' [128][Q <= 16] slice
  static constexpr int RING = B_STAGES * STAGE + A_BUFS * A_RAW;
  static constexpr int SMEM = (RING > EPI ? RING : EPI) + 1024;  // + alignment slack of the 1024-byte swizzle atoms
  // A-fragment register sets (8 registers each) in rotation: FRAG_SETS - 1 of the warpgroup's commit groups stay queued
  // while the next is prepared
  static constexpr int FRAG_SETS = BN == 128 ? 4 : 2;
  // Two CTAs per SM at BN = 64: 128 registers (sm_90a, 0 spills) and 81 KiB (image: 97 KiB) of shared memory each.  One at
  // BN = 128: 223-242 registers, 129 KiB (image: 230 registers, 177 KiB).
  static constexpr int MIN_BLOCKS = BN <= 64 ? 2 : 1;
};

// Epilogue: `stage` holds the raw tile [128][SLD] (sum of both accumulators).  The 256 threads write it out
// row-contiguously, applying bias / ReLU / mask on the way, then run the fused column reductions.
template <int BN>
__device__ __forceinline__ void tile_epilogue(float* stage, const float* s_bias, bool s_bias_on, int m0, int n0, int M, int N,
                                              float* __restrict__ C, int64_t ldc, const TcEpilogue& ep) {
  constexpr int SLD = TileCfg<BN>::SLD;
  constexpr int C4 = BN / 4;
  constexpr int UNR = 4;  // independent row pieces per thread and trip: keeps the mask loads in flight together
  const int rows_here = min(BM, M - m0);
  const int total = rows_here * C4;
  const bool vec_ok = ((ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
  const bool mvec_ok = ep.mask_src && ((ep.ldm & 3) == 0) && ((reinterpret_cast<uintptr_t>(ep.mask_src) & 15) == 0);
  const bool want_hooks = ep.hooks.colsum || ep.hooks.stats || ep.hooks.S;
  for (int base = threadIdx.x; base < total; base += NTHREADS * UNR) {
    float4 o[UNR], mk[UNR];
    int gm[UNR], gn[UNR];
    bool live[UNR];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const int idx = base + u * NTHREADS;
      const int r = idx / C4, c4 = idx - r * C4;
      gm[u] = m0 + r;
      gn[u] = n0 + c4 * 4;
      live[u] = idx < total && gn[u] < N;
      mk[u] = make_float4(1.f, 1.f, 1.f, 1.f);
      if (live[u]) {
        o[u] = *reinterpret_cast<const float4*>(stage + r * SLD + c4 * 4);
        if (ep.mask_src) {
          const float* mp = ep.mask_src + (int64_t)gm[u] * ep.ldm + gn[u];
          if (mvec_ok && gn[u] + 3 < N) mk[u] = *reinterpret_cast<const float4*>(mp);
          else {
            mk[u].x = mp[0];
            mk[u].y = gn[u] + 1 < N ? mp[1] : 1.f;
            mk[u].z = gn[u] + 2 < N ? mp[2] : 1.f;
            mk[u].w = gn[u] + 3 < N ? mp[3] : 1.f;
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      if (!live[u]) continue;
      float ov[4] = {o[u].x, o[u].y, o[u].z, o[u].w};
      const float mv[4] = {mk[u].x, mk[u].y, mk[u].z, mk[u].w};
      const float4 b4 = s_bias_on ? *reinterpret_cast<const float4*>(s_bias + (gn[u] - n0)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (s_bias_on) ov[q] += bv[q];
        if (ep.relu) ov[q] = relu_keep_nan(ov[q]);
        ov[q] = mv[q] > 0.f ? ov[q] : 0.f;
      }
      if (want_hooks)  // keep the final values in the staging tile for the column reductions below
        *reinterpret_cast<float4*>(stage + (gm[u] - m0) * SLD + (gn[u] - n0)) = make_float4(ov[0], ov[1], ov[2], ov[3]);
      float* dst = C + (int64_t)gm[u] * ldc + gn[u];
      if (gn[u] + 3 < N && vec_ok) {
        if (ep.atomic) atomicAdd(reinterpret_cast<float4*>(dst), make_float4(ov[0], ov[1], ov[2], ov[3]));
        else *reinterpret_cast<float4*>(dst) = make_float4(ov[0], ov[1], ov[2], ov[3]);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (gn[u] + q < N) {
            if (ep.atomic) atomicAdd(dst + q, ov[q]); else dst[q] = ov[q];
          }
      }
    }
  }
  // fused column reductions over the final tile: thread c owns output column n0 + c (conflict-free smem column walks),
  // one atomic per (CTA, column[, q])
  if (want_hooks) {
    float* sS = stage + BM * SLD;  // [128][Q] slice of the per-row weights, behind the staging tile
    if (ep.hooks.S)
      for (int i = threadIdx.x; i < rows_here * ep.hooks.Q; i += NTHREADS) sS[i] = ep.hooks.S[(int64_t)m0 * ep.hooks.Q + i];
    __syncthreads();
    const int c = threadIdx.x;
    if (c < BN && n0 + c < N) {
      const int Q = ep.hooks.Q;
      float s1 = 0.f;
      double d1 = 0.0, d2 = 0.0;
      float tq[kMaxHookQ];
#pragma unroll
      for (int q = 0; q < kMaxHookQ; ++q) tq[q] = 0.f;
      for (int r = 0; r < rows_here; ++r) {
        const float v = stage[r * SLD + c];
        s1 += v;
        if (ep.hooks.stats) { d1 += (double)v; d2 += (double)v * (double)v; }
        if (ep.hooks.S) {
#pragma unroll
          for (int q = 0; q < kMaxHookQ; ++q)
            if (q < Q) tq[q] = fmaf(sS[r * Q + q], v, tq[q]);
        }
      }
      if (ep.hooks.colsum) atomicAdd(&ep.hooks.colsum[n0 + c], s1);
      if (ep.hooks.stats) {
        atomicAdd(&ep.hooks.stats[n0 + c], d1);
        atomicAdd(&ep.hooks.stats[(int64_t)N + n0 + c], d2);
      }
      if (ep.hooks.S) {
#pragma unroll
        for (int q = 0; q < kMaxHookQ; ++q)
          if (q < Q)
            atomicAdd(q < ep.hooks.q_split ? &ep.hooks.gT[(int64_t)q * ep.hooks.ldt + n0 + c]
                                           : &ep.hooks.gT2[(int64_t)(q - ep.hooks.q_split) * ep.hooks.ldt + n0 + c], tq[q]);
      }
    }
  }
}

// C[m, n] = sum_r A(m, r) * B(n, r) over r in [kbeg, kend) of this split (split z stores at C + z * ep.split_stride).  B_IMG: B is
// the hi plane of a weight image (row stride ldb = img_ld(K), lo plane img_rows(N) rows behind it), K-major A and B only.
template <bool A_KC, bool B_KC, int BN, bool B_IMG>
__global__ void __launch_bounds__(NTHREADS, TileCfg<BN, B_IMG>::MIN_BLOCKS)
k_gemm_3xtf32(const float* __restrict__ A, int64_t lda, const float* __restrict__ B, int64_t ldb, float* __restrict__ C, int64_t ldc,
              int M, int N, int K, int k_per_split, TcEpilogue ep) {
  static_assert(BN == 64 || BN == 128, "one wgmma.m64nBNk8 per product; two accumulators of BN / 2 registers each");
  static_assert(!B_IMG || (A_KC && B_KC), "the image path serves the forward and dgrad GEMMs: K-major A and B");
  using Cfg = TileCfg<BN, B_IMG>;
  constexpr int NF = Cfg::FRAG_SETS;
  constexpr int NB = Cfg::B_STAGES, NA = Cfg::A_BUFS;
  static_assert((BK / 8) % NF == 0, "k-step j uses fragment set j % NF in every block");
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(16) float s_bias[BN];
  // the swizzle pattern is a function of the address bits: stages start on 1024-byte boundaries
  uint8_t* smem = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
  auto b_hi = [&](int s) { return smem + s * Cfg::STAGE; };
  auto b_lo = [&](int s) { return b_hi(s) + Cfg::B_BYTES; };
  float* a_raw = reinterpret_cast<float*>(smem + NB * Cfg::STAGE);  // NA raw A blocks

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int t = lane & 3;
  const int mrow = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's A-fragment rows: mrow and mrow + 8
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);
  const int nkb = (kend - kbeg + BK - 1) / BK;
  const bool s_bias_on = ep.bias != nullptr && blockIdx.z == 0;

  pdl_prologue();
  for (int i = threadIdx.x; i < BN; i += NTHREADS) s_bias[i] = (s_bias_on && n0 + i < N) ? ep.bias[n0 + i] : 0.f;

  Loader<B_KC, BN> lb;  // raw B only: unused (and without registers) in the image instantiations
  if constexpr (!B_IMG) lb.init(B, ldb, n0, N, kbeg);
  const int64_t plane = B_IMG ? img_rows(N) * ldb : 0;  // image: hi plane -> lo plane

  float acc[BN / 2], accx[BN / 2];  // hi*hi chain | cross terms
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = accx[i] = 0.f;
  uint32_t fh[NF][4], fl[NF][4];  // A fragment hi / lo, NF sets

  if (nkb > 0) {
    a_copy<A_KC>(a_raw, A, lda, m0, M, kbeg, kend - kbeg);
    if constexpr (B_IMG) {
      // commit groups: {A 0, B 0}, {A 1 when two ahead, B 1}; then one group per block (two when A is one ahead, A first), so
      // that after wait_group 1 only the newest, block kb + 2's B, may still be in flight
      b_img_copy<BN>(b_hi(0), b_lo(0), B, ldb, plane, n0, kbeg);
      cp_async_commit();
      if (nkb > 1) {
        if (Cfg::A_DIST == 2) a_copy<A_KC>(a_raw + BM * BK, A, lda, m0, M, kbeg + BK, kend - kbeg - BK);
        b_img_copy<BN>(b_hi(1), b_lo(1), B, ldb, plane, n0, kbeg + BK);
      }
      cp_async_commit();
      cp_async_wait<1>();
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // cp.async writes the generic proxy: -> the tensor cores
    } else {
      cp_async_commit();
      lb.load(0, kend - kbeg);
      lb.store(b_hi(0), b_lo(0));
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the tensor cores
      cp_async_wait_all();
    }
  }
  int s = 0, sa = 0;  // B stage and (image path) A buffer of block kb; the raw path's A buffer is kb & 1
#pragma unroll 1
  for (int kb = 0; kb < nkb; ++kb) {
    // B stage s and A buffer sa are complete.  Every thread has retired its warpgroup's groups of block kb - 2 (at most NF - 1
    // groups are in flight after a wait), so B stage (kb - 2) mod NB is free: for block kb + 1 with NB = 3 stages, kb + 2 with
    // four.  A buffer (kb - 1) mod NA was read by block kb - 1's fragment loads: block kb + NA - 1 goes there.
    __syncthreads();
    const bool more = kb + 1 < nkb;
    if constexpr (B_IMG) {  // copies of block kb + 2 (and of A kb + 1 when it is one ahead) fly under this block's MMAs
      if (Cfg::A_DIST == 1) {
        const int k1 = kbeg + (kb + 1) * BK;
        if (more) a_copy<A_KC>(a_raw + (sa ^ 1) * (BM * BK), A, lda, m0, M, k1, kend - k1);
        cp_async_commit();
      }
      if (kb + 2 < nkb) {
        const int k2 = kbeg + (kb + 2) * BK, s2 = s + 2 < NB ? s + 2 : s + 2 - NB;
        if (Cfg::A_DIST == 2) a_copy<A_KC>(a_raw + (sa == 0 ? NA - 1 : sa - 1) * (BM * BK), A, lda, m0, M, k2, kend - k2);
        b_img_copy<BN>(b_hi(s2), b_lo(s2), B, ldb, plane, n0, k2);
      }
      cp_async_commit();  // possibly empty: every block commits the same number of groups
    } else if (more) {  // next block's copies and global loads fly under this block's MMAs
      a_copy<A_KC>(a_raw + ((kb + 1) & 1) * (BM * BK), A, lda, m0, M, kbeg + (kb + 1) * BK, kend - kbeg - (kb + 1) * BK);
      cp_async_commit();
      lb.load(kb + 1, kend - kbeg - (kb + 1) * BK);
    }
    const float* ar = a_raw + (B_IMG ? sa : kb & 1) * (BM * BK);
    float4 av[2];  // K-major A: elements 16 (j / 2) + 4t .. + 3 of rows mrow, mrow + 8 (the slots of k-steps j, j + 1 for even j)
    const uint64_t dh = gmma_desc_sw128(smem_u32(b_hi(s))), dl = gmma_desc_sw128(smem_u32(b_lo(s)));
#pragma unroll
    for (int j = 0; j < BK / 8; ++j) {  // k-step j: 8 fp32 = 32 bytes into the 128-byte swizzle row
      const int f = j % NF;
      wgmma_wait<NF - 1>();  // the group that last read set f (k-step j - NF) has retired
      if (A_KC && (j & 1) == 0) {
#pragma unroll
        for (int r = 0; r < 2; ++r) av[r] = *reinterpret_cast<const float4*>(ar + akc_off(mrow + 8 * r, 16 * (j >> 1) + 4 * t));
      }
      float x[4];  // fragment rows mrow, mrow + 8 at columns t, t + 4 of the k-step
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int slot = 2 * (j & 1) + (q >> 1);  // element of the thread's 4-element piece
        if (A_KC) x[q] = f4_at(av[q & 1], slot);
        else x[q] = ar[araw_off(mrow + 8 * (q & 1), 16 * (j >> 1) + 4 * t + slot)];
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float h, l;
        split_tf32(x[q], h, l);
        fh[f][q] = __float_as_uint(h);
        fl[f][q] = __float_as_uint(l);
      }
      wgmma_fence();
      wgmma_tf32_rs<BN>(accx, fl[f], dh + 2 * j);  // + j * 32 bytes in the descriptor's 16-byte address units
      wgmma_tf32_rs<BN>(accx, fh[f], dl + 2 * j);
      wgmma_tf32_rs<BN>(acc, fh[f], dh + 2 * j);
      wgmma_commit();
    }
    s = s + 1 == NB ? 0 : s + 1;
    if constexpr (B_IMG) sa = sa + 1 == NA ? 0 : sa + 1;
    if (more) {
      if constexpr (B_IMG) {
        cp_async_wait<1>();  // this thread's copies of block kb + 1 have landed (block kb + 2's B may still fly)
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      } else {
        lb.store(b_hi(s), b_lo(s));
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        cp_async_wait_all();  // this thread's A copies of block kb + 1 have landed; the barrier publishes them
      }
    }
  }
  if constexpr (B_IMG) cp_async_wait_all();  // only empty groups can be left; nothing may land in the staging tile
  wgmma_wait<0>();
  fence_acc(acc);
  fence_acc(accx);
  __syncthreads();  // the stages are free: the staging tile reuses them

  // accumulator fragment of wgmma m64nN (f32): register 4i + j of lane l in warp w of the warpgroup holds
  // row 16 w + l / 4 + 8 (j / 2), column 8 i + 2 (l % 4) + (j % 2)
  float* stage = reinterpret_cast<float*>(smem);
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
    const int col = i * 8 + t * 2;
    *reinterpret_cast<float2*>(stage + mrow * Cfg::SLD + col) =
        make_float2(sum_chains(acc[4 * i], accx[4 * i]), sum_chains(acc[4 * i + 1], accx[4 * i + 1]));
    *reinterpret_cast<float2*>(stage + (mrow + 8) * Cfg::SLD + col) =
        make_float2(sum_chains(acc[4 * i + 2], accx[4 * i + 2]), sum_chains(acc[4 * i + 3], accx[4 * i + 3]));
  }
  __syncthreads();
  tile_epilogue<BN>(stage, s_bias, s_bias_on, m0, n0, M, N, C + (int64_t)blockIdx.z * ep.split_stride, ldc, ep);
}

// gb[n] = sum_m gy[m][n]: 32 columns x 8 row-lanes per block, coalesced row sweeps, smem fold, one atomic per column
__global__ void __launch_bounds__(256)
k_colsum_tc(const float* __restrict__ gy, int64_t ld, int M, int N, int rows_per_block, float* __restrict__ gb) {
  pdl_prologue();
  __shared__ float red[8][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + lane;
  const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
  float a = 0.f;
  if (n < N) {
#pragma unroll 4
    for (int r = r0 + w; r < r1; r += 8) a += gy[(int64_t)r * ld + n];
  }
  red[w][lane] = a;
  __syncthreads();
  if (w == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][lane];
    atomicAdd(&gb[n], t);
  }
}

template <bool A_KC, bool B_KC, int BN, bool B_IMG = false>
int launch(const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int M, int N, int K, int splits,
           int k_per_split, const TcEpilogue& ep, cudaStream_t st) {
  constexpr int smem = TileCfg<BN, B_IMG>::SMEM;
  // the shared-memory opt-in belongs to the current device's context: set it once per device (bit d = device d)
  static std::atomic<uint64_t> configured{0};
  int dev = 0;
  PGNN_CUDA(cudaGetDevice(&dev));
  const uint64_t bit = dev < 64 ? (uint64_t)1 << dev : 0;
  if (!(configured.load(std::memory_order_relaxed) & bit)) {
    PGNN_CUDA(cudaFuncSetAttribute(k_gemm_3xtf32<A_KC, B_KC, BN, B_IMG>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured.fetch_or(bit, std::memory_order_relaxed);
  }
  dim3 grid((unsigned)ceil_div(N, BN), (unsigned)ceil_div(M, BM), (unsigned)splits);
  PGNN_CUDA(pgnn_launch(k_gemm_3xtf32<A_KC, B_KC, BN, B_IMG>, dim3(grid), dim3(NTHREADS), smem, st, A, lda, B, ldb, C, ldc, M, N, K, k_per_split, ep));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

// Tile width: the one with the least per-SM work over the whole grid, waves x (BN x CTAs resident per SM); a BN = 64
// CTA holds half the shared memory and registers of a BN = 128 one, so two of them share an SM.  Ties go to the wider
// tile (fewer re-reads of the A rows).
inline int pick_bn(int M, int N, int splits) {
  const int64_t mt = ceil_div(M, BM) * (splits > 0 ? splits : 1);
  auto cost = [&](int bn, int per_sm) { return ceil_div(mt * ceil_div(N, bn), (int64_t)kNumSMs * per_sm) * bn * per_sm; };
  return cost(64, TileCfg<64>::MIN_BLOCKS) < cost(128, TileCfg<128>::MIN_BLOCKS) ? 64 : 128;
}

template <bool A_KC, bool B_KC>
int dispatch(int bn, const float* A, int64_t lda, const float* B, int64_t ldb, float* C, int64_t ldc, int M, int N, int K, int splits,
             int k_per_split, const TcEpilogue& ep, cudaStream_t st) {
  if (ep.hooks.S && (ep.hooks.Q < 1 || ep.hooks.Q > kMaxHookQ)) return PGNN_EINVAL;
  if (bn == 64) return launch<A_KC, B_KC, 64>(A, lda, B, ldb, C, ldc, M, N, K, splits, k_per_split, ep, st);
  return launch<A_KC, B_KC, 128>(A, lda, B, ldb, C, ldc, M, N, K, splits, k_per_split, ep, st);
}

// C[M, N] = A[M, K] . B^T from the weight image `img` of B (hi plane first, img_ld(K) floats per row), one split
int dispatch_img(int bn, const float* A, int64_t lda, const float* img, float* C, int64_t ldc, int M, int N, int K, const TcEpilogue& ep,
                 cudaStream_t st) {
  if (ep.hooks.S && (ep.hooks.Q < 1 || ep.hooks.Q > kMaxHookQ)) return PGNN_EINVAL;
  if (bn == 64) return launch<true, true, 64, true>(A, lda, img, img_ld(K), C, ldc, M, N, K, 1, K, ep, st);
  return launch<true, true, 128, true>(A, lda, img, img_ld(K), C, ldc, M, N, K, 1, K, ep, st);
}

// Weight images (see img_rows above) for a batch of weights: job j reads w[rows][cols] (row stride ld) and writes the image of w as
// a K-major B (B rows = rows, reduction = cols) or, transposed, of w^T (B rows = cols, reduction = rows).  One CTA per 32 x 32 piece
// of the image; the piece goes through shared memory so that both source orientations are read along their contiguous extent.
struct PackJob { const float* w; float* img; int64_t ld; int rows, cols, trans; };
constexpr int kMaxPackJobs = 32;
struct PackBatch { PackJob job[kMaxPackJobs]; };
__global__ void __launch_bounds__(256) k_pack_img_batch(PackBatch b) {
  pdl_prologue();
  __shared__ float tile[32][33];  // [image row][reduction index]
  const PackJob j = b.job[blockIdx.z];
  const int R = j.trans ? j.cols : j.rows, Kr = j.trans ? j.rows : j.cols;
  const int64_t ld = img_ld(Kr), nr = img_rows(R);
  const int k0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  if (k0 >= ld || r0 >= nr) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    if (j.trans) {  // w^T: image row r0 + tx is column r0 + tx of w
      const int r = r0 + tx, k = k0 + i;
      tile[tx][i] = r < R && k < Kr ? j.w[(int64_t)k * j.ld + r] : 0.f;
    } else {
      const int r = r0 + i, k = k0 + tx;
      tile[i][tx] = r < R && k < Kr ? j.w[(int64_t)r * j.ld + k] : 0.f;
    }
  }
  __syncthreads();
  const int rr = threadIdx.x >> 3, c = (threadIdx.x & 7) * 4;  // one 16-byte piece (slots c .. c + 3) of row r0 + rr per plane
  float h[4], l[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) split_tf32(tile[rr][kperm(c + q)], h[q], l[q]);
  float* dst = j.img + (int64_t)(r0 + rr) * ld + k0 + c;
  *reinterpret_cast<float4*>(dst) = make_float4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<float4*>(dst + nr * ld) = make_float4(l[0], l[1], l[2], l[3]);
}

}  // namespace

// floats of the weight image of a K-major B with `rows` rows and reduction k (both planes)
int64_t pgnn_tc_image_floats(int64_t rows, int64_t k) { return 2 * img_rows(rows) * img_ld(k); }

// count <= 32 weight images in one launch (PackJob above; rows, cols of the SOURCE w)
int pgnn_internal_pack_images(int count, const float* const* w, const int64_t* ld, const int* rows, const int* cols, const int* trans,
                              float* const* img, cudaStream_t st) {
  if (count <= 0) return PGNN_OK;
  if (count > kMaxPackJobs) return PGNN_EUNSUPPORTED;
  PackBatch b;
  int64_t mr = 0, mk = 0;
  for (int i = 0; i < count; ++i) {
    if (!aligned16(img[i])) return PGNN_EUNSUPPORTED;
    b.job[i] = PackJob{w[i], img[i], ld[i], rows[i], cols[i], trans[i] ? 1 : 0};
    const int64_t R = img_rows(trans[i] ? cols[i] : rows[i]), K = img_ld(trans[i] ? rows[i] : cols[i]);
    mr = R > mr ? R : mr;
    mk = K > mk ? K : mk;
  }
  dim3 grid((unsigned)(mk / 32), (unsigned)(mr / 32), (unsigned)count);
  PGNN_CUDA(pgnn_launch(k_pack_img_batch, dim3(grid), dim3(256), 0, st, b));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

// The forward and dgrad GEMMs from a weight image (pgnn_internal_pack_images): img_rows / img_k = the image's padded row count and
// row stride, which must be img_rows(output columns) and img_ld(reduction).  Same epilogues as the raw-weight entry points.
// y[M,N] = act(x[M,K] . w[N,K]^T + bias), img = the image of w
int pgnn_tc_linear_fwd_img(const float* x, int64_t ldx, const float* img, int64_t img_r, int64_t img_k, const float* bias, int64_t M,
                           int64_t N, int64_t K, int relu, float* y, int64_t ldy, cudaStream_t st, const PgnnGemmHooks* hooks) {
  if (img_r != img_rows(N) || img_k != img_ld(K)) return PGNN_EINVAL;
  if (ldx % 4 || !aligned16(x) || !aligned16(img) || !aligned16(y) || M < 1) return PGNN_EUNSUPPORTED;
  TcEpilogue ep{bias, relu, nullptr, 0, 0, hooks ? *hooks : PgnnGemmHooks{}};
  return dispatch_img(pick_bn((int)M, (int)N, 1), x, ldx, img, y, ldy, (int)M, (int)N, (int)K, ep, st);
}

// gx[M,K] = (gy[M,N] . w[N,K]) masked by relu_src > 0, img = the image of w^T (B rows K, reduction N)
int pgnn_tc_linear_bwd_x_img(const float* gy, int64_t ldgy, const float* img, int64_t img_r, int64_t img_k, int64_t M, int64_t N,
                             int64_t K, const float* relu_src, int64_t ldr, float* gx, int64_t ldgx, cudaStream_t st,
                             const PgnnGemmHooks* hooks) {
  if (img_r != img_rows(K) || img_k != img_ld(N)) return PGNN_EINVAL;
  if (ldgy % 4 || !aligned16(gy) || !aligned16(img) || !aligned16(gx) || M < 1) return PGNN_EUNSUPPORTED;
  TcEpilogue ep{nullptr, 0, relu_src, ldr, 0, hooks ? *hooks : PgnnGemmHooks{}};
  return dispatch_img(pick_bn((int)M, (int)K, 1), gy, ldgy, img, gx, ldgx, (int)M, (int)K, (int)N, ep, st);
}

extern "C" int pgnn_debug_pack_weight_images(int count, const float* const* w, const int64_t* ld, const int32_t* rows,
                                             const int32_t* cols, const int32_t* transposed, float* const* img, void* stream) {
  PGNN_CHECK_ARG(count >= 0);
  if (count == 0) return PGNN_OK;
  PGNN_CHECK_ARG(w && ld && rows && cols && transposed && img);
  if (count > kMaxPackJobs) return PGNN_EUNSUPPORTED;
  for (int i = 0; i < count; ++i) PGNN_CHECK_ARG(w[i] && img[i] && rows[i] > 0 && cols[i] > 0 && ld[i] >= cols[i]);
  return pgnn_internal_pack_images(count, w, ld, rows, cols, transposed, img, as_stream(stream));
}

namespace {
// the epilogue arguments of the two GEMM test entry points
int debug_epilogue(int64_t N, const float* bias, int relu, const float* mask, int64_t ldm, float* colsum, double* stats, const float* S,
                   int Q, float* gT, float* gT2, int q_split, int64_t ldt, TcEpilogue& ep) {
  PGNN_CHECK_ARG(!mask || ldm >= N);
  if (S) {
    PGNN_CHECK_ARG(Q >= 1 && Q <= kMaxHookQ && q_split >= 0 && q_split <= Q && ldt >= N);
    PGNN_CHECK_ARG((q_split == 0 || gT) && (q_split == Q || gT2));
  }
  ep = TcEpilogue{bias, relu, mask, ldm, 0, PgnnGemmHooks{}};
  ep.hooks.colsum = colsum;
  ep.hooks.stats = stats;
  ep.hooks.S = S;
  ep.hooks.Q = S ? Q : 0;
  ep.hooks.gT = gT;
  ep.hooks.gT2 = gT2;
  ep.hooks.q_split = q_split;
  ep.hooks.ldt = ldt;
  return PGNN_OK;
}
}  // namespace

extern "C" int pgnn_debug_tc_gemm_img(int bn, const float* A, int64_t lda, const float* B, int64_t ldb, float* img, float* C, int64_t ldc,
                                      int64_t M, int64_t N, int64_t K, const float* bias, int relu, const float* mask, int64_t ldm,
                                      float* colsum, double* stats, const float* S, int Q, float* gT, float* gT2, int q_split,
                                      int64_t ldt, void* stream) {
  PGNN_CHECK_ARG(bn == 64 || bn == 128);
  PGNN_CHECK_ARG(M > 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31));
  PGNN_CHECK_ARG(A && B && img && C && ldc >= N && lda >= K && ldb >= K);
  TcEpilogue ep;
  const int rc = debug_epilogue(N, bias, relu, mask, ldm, colsum, stats, S, Q, gT, gT2, q_split, ldt, ep);
  if (rc != PGNN_OK) return rc;
  if (lda % 4 || ldb % 4 || !aligned16(A) || !aligned16(B) || !aligned16(img)) return PGNN_EUNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  const int r = (int)N, c = (int)K, zero = 0;
  const int prc = pgnn_internal_pack_images(1, &B, &ldb, &r, &c, &zero, &img, st);
  if (prc != PGNN_OK) return prc;
  return dispatch_img(bn, A, lda, img, C, ldc, (int)M, (int)N, (int)K, ep, st);
}

extern "C" int pgnn_debug_tc_gemm(int a_kc, int b_kc, int bn, const float* A, int64_t lda, const float* B, int64_t ldb, float* C,
                                  int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias, int relu, const float* mask,
                                  int64_t ldm, float* colsum, double* stats, const float* S, int Q, float* gT, float* gT2,
                                  int q_split, int64_t ldt, void* stream) {
  PGNN_CHECK_ARG(bn == 64 || bn == 128);
  PGNN_CHECK_ARG(M > 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31));
  PGNN_CHECK_ARG(A && B && C && ldc >= N && lda >= (a_kc ? K : M) && ldb >= (b_kc ? K : N));
  TcEpilogue ep;
  const int rc = debug_epilogue(N, bias, relu, mask, ldm, colsum, stats, S, Q, gT, gT2, q_split, ldt, ep);
  if (rc != PGNN_OK) return rc;
  if (lda % 4 || ldb % 4 || !aligned16(A) || !aligned16(B)) return PGNN_EUNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  const int m = (int)M, n = (int)N, k = (int)K;
  if (a_kc && b_kc) return dispatch<true, true>(bn, A, lda, B, ldb, C, ldc, m, n, k, 1, k, ep, st);
  if (a_kc && !b_kc) return dispatch<true, false>(bn, A, lda, B, ldb, C, ldc, m, n, k, 1, k, ep, st);
  if (!a_kc && b_kc) return dispatch<false, true>(bn, A, lda, B, ldb, C, ldc, m, n, k, 1, k, ep, st);
  return dispatch<false, false>(bn, A, lda, B, ldb, C, ldc, m, n, k, 1, k, ep, st);
}

// y[M,N] = act(x[M,K] . w[N,K]^T + bias)
int pgnn_tc_linear_fwd(const float* x, int64_t ldx, const float* w, const float* bias, int64_t M, int64_t N, int64_t K, int relu,
                       float* y, int64_t ldy, cudaStream_t st, const PgnnGemmHooks* hooks) {
  if (K % 4 || ldx % 4 || !aligned16(x) || !aligned16(w) || !aligned16(y) || M < 1) return PGNN_EUNSUPPORTED;
  TcEpilogue ep{bias, relu, nullptr, 0, 0, hooks ? *hooks : PgnnGemmHooks{}};
  return dispatch<true, true>(pick_bn((int)M, (int)N, 1), x, ldx, w, K, y, ldy, (int)M, (int)N, (int)K, 1, (int)K, ep, st);
}

// gx[M,K] = (gy[M,N] . w[N,K]) masked by relu_src > 0
int pgnn_tc_linear_bwd_x(const float* gy, int64_t ldgy, const float* w, int64_t M, int64_t N, int64_t K, const float* relu_src,
                         int64_t ldr, float* gx, int64_t ldgx, cudaStream_t st, const PgnnGemmHooks* hooks) {
  if (K % 4 || ldgy % 4 || !aligned16(gy) || !aligned16(w) || !aligned16(gx) || M < 1) return PGNN_EUNSUPPORTED;
  TcEpilogue ep{nullptr, 0, relu_src, ldr, 0, hooks ? *hooks : PgnnGemmHooks{}};
  // output columns are K; the reduction runs over N; B(n_out = k, r = n) = w[r*K + k] is row-index contiguous
  return dispatch<true, false>(pick_bn((int)M, (int)K, 1), gy, ldgy, w, K, gx, ldgx, (int)M, (int)K, (int)N, 1, (int)N, ep, st);
}

// out[c][r] = in[r][c] for a batch of row-major matrices (weights: a few hundred KB each)
namespace {
struct TransposeJob { const float* in; float* out; int rows, cols; };
constexpr int kMaxTransposeJobs = 32;
struct TransposeBatch { TransposeJob job[kMaxTransposeJobs]; };
__global__ void __launch_bounds__(256) k_transpose_batch(TransposeBatch b) {
  pdl_prologue();
  __shared__ float tile[32][33];
  const TransposeJob j = b.job[blockIdx.z];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  if (c0 >= j.cols || r0 >= j.rows) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8)
    if (r0 + i < j.rows && c0 + tx < j.cols) tile[i][tx] = j.in[(int64_t)(r0 + i) * j.cols + c0 + tx];
  __syncthreads();
  for (int i = ty; i < 32; i += 8)
    if (c0 + i < j.cols && r0 + tx < j.rows) j.out[(int64_t)(c0 + i) * j.rows + r0 + tx] = tile[tx][i];
}
}  // namespace

int pgnn_internal_transpose_batch(int count, const float* const* in, float* const* out, const int* rows, const int* cols,
                                  cudaStream_t st) {
  if (count <= 0) return PGNN_OK;
  if (count > kMaxTransposeJobs) return PGNN_EUNSUPPORTED;
  TransposeBatch b;
  int mr = 0, mc = 0;
  for (int i = 0; i < count; ++i) {
    b.job[i] = TransposeJob{in[i], out[i], rows[i], cols[i]};
    mr = rows[i] > mr ? rows[i] : mr;
    mc = cols[i] > mc ? cols[i] : mc;
  }
  dim3 grid((unsigned)ceil_div(mc, 32), (unsigned)ceil_div(mr, 32), (unsigned)count);
  PGNN_CUDA(pgnn_launch(k_transpose_batch, dim3(grid), dim3(256), 0, st, b));
  PGNN_LAUNCH_CHECK();
  return PGNN_OK;
}

namespace {
// out[i] = sum_s part[s][i]: folds the split-K partial tiles (plain coalesced stores from the GEMM epilogue instead of
// vector atomics on the same 0.7 MB of output)
__global__ void __launch_bounds__(256) k_splitk_reduce(const float* __restrict__ part, int splits, int64_t n4, float* __restrict__ out) {
  pdl_prologue();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4* p = reinterpret_cast<const float4*>(part) + i;
    float4 a = p[0];
    int s = 1;
    for (; s + 3 < splits; s += 4) {  // four independent loads in flight; the sum order stays s = 0, 1, 2, ... (deterministic)
      const float4 b0 = p[(int64_t)s * n4], b1 = p[(int64_t)(s + 1) * n4], b2 = p[(int64_t)(s + 2) * n4], b3 = p[(int64_t)(s + 3) * n4];
      a.x += b0.x; a.y += b0.y; a.z += b0.z; a.w += b0.w;
      a.x += b1.x; a.y += b1.y; a.z += b1.z; a.w += b1.w;
      a.x += b2.x; a.y += b2.y; a.z += b2.z; a.w += b2.w;
      a.x += b3.x; a.y += b3.y; a.z += b3.z; a.w += b3.w;
    }
    for (; s < splits; ++s) {
      const float4 b = p[(int64_t)s * n4];
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    reinterpret_cast<float4*>(out)[i] = a;
  }
}

// tile width, split count and rows per split of the weight-gradient GEMM gw[N,K] = gy[M,N]^T . x[M,K]
struct WgradPlan { int bn, tiles, splits, per; };
WgradPlan wgrad_plan(int64_t M, int64_t N, int64_t K) {
  WgradPlan p;
  p.bn = 128;  // the reduction is long and both operands are re-read per tile: the wider tile unless it pads > 15%
  if ((int)ceil_div(K, 128) * 128 > K + K * 15 / 100) p.bn = 64;
  p.tiles = (int)(ceil_div(N, BM) * ceil_div(K, p.bn));
  int splits = kNumSMs * TileCfg<128>::MIN_BLOCKS / p.tiles;  // floor: one more CTA than the chip holds would be a second wave
  if (p.bn == 64) splits = kNumSMs * TileCfg<64>::MIN_BLOCKS / p.tiles;
  // keep each accumulation chain <= 1024 rows, fold the rest in fp32
  if (splits < (int)ceil_div(M, 1024)) splits = (int)ceil_div(M, 1024);
  const int max_splits = (int)ceil_div(M, 2 * BK);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  p.per = (int)align_up(ceil_div(M, splits), BK);
  p.splits = (int)ceil_div(M, p.per);
  return p;
}
}  // namespace

// floats of split-K workspace pgnn_tc_linear_bwd_w_ws needs for this problem: one partial tile set per split
int64_t pgnn_tc_wgrad_workspace_floats(int64_t M, int64_t N, int64_t K) {
  if (M < 1) M = 1;
  const WgradPlan p = wgrad_plan(M, N, K);
  return (int64_t)p.splits * N * K;
}

// gw[N,K] = gy[M,N]^T . x[M,K]; gb[N] = column sums of gy.  `partials` (optional, >= splits*N*K floats): split-K partial
// tiles are stored there and folded by one reduction kernel; without it the epilogue uses vector atomics.
int pgnn_tc_linear_bwd_w_ws(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t N, int64_t K, float* gw,
                            float* gb, float* partials, int64_t partial_floats, cudaStream_t st) {
  if (K % 4 || ldgy % 4 || ldx % 4 || !aligned16(gy) || !aligned16(x) || !aligned16(gw) || M < 1) return PGNN_EUNSUPPORTED;
  // output [N, K] (rows N = "M" of the MMA), reduction over the M node rows, split so the grid fills the chip
  const WgradPlan plan = wgrad_plan(M, N, K);
  const int bn = plan.bn, splits = plan.splits, per = plan.per;
  int rc;
  if (splits > 1 && partials && aligned16(partials) && partial_floats >= (int64_t)splits * N * K && ((N * K) % 4 == 0)) {
    // split s writes its tile into partials[s] (the kernel offsets C by blockIdx.z * ep.split_stride)
    TcEpilogue ep{nullptr, 0, nullptr, 0, 0, PgnnGemmHooks{}};
    ep.split_stride = N * K;
    rc = dispatch<false, false>(bn, gy, ldgy, x, ldx, partials, K, (int)N, (int)K, (int)M, splits, per, ep, st);
    if (rc != PGNN_OK) return rc;
    const int64_t n4 = N * K / 4;
    int blocks = (int)ceil_div(n4, 256);
    if (blocks > kNumSMs * 4) blocks = kNumSMs * 4;
    PGNN_CUDA(pgnn_launch(k_splitk_reduce, dim3(blocks), dim3(256), 0, st, partials, splits, n4, gw));
    PGNN_LAUNCH_CHECK();
  } else {
    if (splits > 1) PGNN_CUDA(cudaMemsetAsync(gw, 0, sizeof(float) * N * K, st));
    TcEpilogue ep{nullptr, 0, nullptr, 0, splits > 1, PgnnGemmHooks{}};
    rc = dispatch<false, false>(bn, gy, ldgy, x, ldx, gw, K, (int)N, (int)K, (int)M, splits, per, ep, st);
    if (rc != PGNN_OK) return rc;
  }
  if (gb) {
    PGNN_CUDA(cudaMemsetAsync(gb, 0, sizeof(float) * N, st));
    const int rows_per = M >= 16384 ? 256 : 64;  // 8 rows per thread for small batches: the row loop is a latency chain
    dim3 g2((unsigned)ceil_div(N, 32), (unsigned)ceil_div(M, rows_per));
    PGNN_CUDA(pgnn_launch(k_colsum_tc, dim3(g2), dim3(256), 0, st, gy, ldgy, (int)M, (int)N, rows_per, gb));
    PGNN_LAUNCH_CHECK();
  }
  return PGNN_OK;
}

int pgnn_tc_linear_bwd_w(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t N, int64_t K, float* gw,
                         float* gb, cudaStream_t st) {
  return pgnn_tc_linear_bwd_w_ws(gy, ldgy, x, ldx, M, N, K, gw, gb, nullptr, 0, st);
}

// test entry points (include/pgnn_b200.h): the weight-gradient GEMM with a caller-chosen split-K workspace, its plan, and the
// batched transpose
extern "C" {

int pgnn_debug_tc_wgrad(const float* gy, int64_t ldgy, const float* x, int64_t ldx, int64_t M, int64_t N, int64_t K, float* gw,
                        float* gb, float* partials, int64_t partial_floats, void* stream) {
  PGNN_CHECK_ARG(M > 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31));
  PGNN_CHECK_ARG(gy && x && gw && ldgy >= N && ldx >= K && partial_floats >= 0);
  return pgnn_tc_linear_bwd_w_ws(gy, ldgy, x, ldx, M, N, K, gw, gb, partials, partial_floats, as_stream(stream));
}

int pgnn_debug_tc_wgrad_plan(int64_t M, int64_t N, int64_t K, int64_t* out4) {
  PGNN_CHECK_ARG(M > 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31) && out4);
  const WgradPlan p = wgrad_plan(M, N, K);
  out4[0] = p.bn;
  out4[1] = p.tiles;
  out4[2] = p.splits;
  out4[3] = p.per;
  return PGNN_OK;
}

int pgnn_debug_transpose_batch(int count, const float* const* in, float* const* out, const int32_t* rows, const int32_t* cols,
                               void* stream) {
  PGNN_CHECK_ARG(count >= 0);
  if (count == 0) return PGNN_OK;
  PGNN_CHECK_ARG(in && out && rows && cols);
  if (count > kMaxTransposeJobs) return PGNN_EUNSUPPORTED;
  for (int i = 0; i < count; ++i) PGNN_CHECK_ARG(in[i] && out[i] && rows[i] > 0 && cols[i] > 0);
  return pgnn_internal_transpose_batch(count, in, out, rows, cols, as_stream(stream));
}

}  // extern "C"
