// kernels.cu -- HBM-bound kernels of the N-pair hot path (everything except the two tensor-core contractions).
// Each kernel cites the reference code it replaces (paths relative to /root/reference).
#include <cassert>
#include <cstdlib>
#include "kernels.cuh"
#include <cuda.h>

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cfloat>

#include "thresholds.cuh"   // f2ord / ord2f come with kernels.cuh

namespace npair {
unsigned long long g_kernel_launches = 0;


// --------------------------------------------------------------------------------------------
// small helpers
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// split an fp32 value into 2-byte pieces (see gemm_wgmma.cuh header)
template <int PREC>
__device__ __forceinline__ void split3(float v, uint16_t& p0, uint16_t& p1, uint16_t& p2) {
  if (PREC == PREC_BF16) {
    p0 = __bfloat16_as_ushort(__float2bfloat16_rn(v)); p1 = 0; p2 = 0;
  } else if (PREC == PREC_FP16X2) {
    const __half h = __float2half_rn(v);
    const float r = v - __half2float(h);
    p0 = __half_as_ushort(h); p1 = __half_as_ushort(__float2half_rn(r)); p2 = 0;
  } else {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    const float r1 = v - __bfloat162float(h);
    const __nv_bfloat16 m = __float2bfloat16_rn(r1);
    const float r2 = r1 - __bfloat162float(m);
    p0 = __bfloat16_as_ushort(h); p1 = __bfloat16_as_ushort(m); p2 = __bfloat16_as_ushort(__float2bfloat16_rn(r2));
  }
}
// Eight consecutive features v, times the pre-scale sc, as pieces: p[e][s] is piece s of feature e, pk[s] the eight pieces s packed into
// one 16-byte group (only the format's pieces are packed)
template <int PREC>
__device__ __forceinline__ void split8(const float (&v)[8], float sc, uint16_t (&p)[8][3], uint4 (&pk)[3]) {
#pragma unroll
  for (int e = 0; e < 8; ++e) split3<PREC>(v[e] * sc, p[e][0], p[e][1], p[e][2]);
#pragma unroll
  for (int s = 0; s < SPLIT_FORMATS[PREC].pieces; ++s)
    pk[s] = make_uint4(p[0][s] | (static_cast<uint32_t>(p[1][s]) << 16), p[2][s] | (static_cast<uint32_t>(p[3][s]) << 16),
                       p[4][s] | (static_cast<uint32_t>(p[5][s]) << 16), p[6][s] | (static_cast<uint32_t>(p[7][s]) << 16));
}
// The packed pieces pk of features [d, d + 8) into one row of the K-concatenated operands of the bitwise-symmetric similarity GEMM,
// in the A (side_b = false) or B format; one Dp-long segment per MMA pass:
//   bf16   : A row = B row = [ hi ]                                                                                       K_cat = Dp
//   fp16x2 : A row = [ hi | hi(8) lo(8) ... ]                         B row = [ hi | lo(8) hi(8) ... ]                  K_cat = 3*Dp
//   bf16x3 : A row = [ hi | mid | hi(8) mid(8) ... | hi(8) lo(8) ... ]   B row = [ hi | mid | mid(8) hi(8) ... | lo(8) hi(8) ... ]   K_cat = 6*Dp
// ONE K=16 MMA then sums 8 products p_j*q_m and the 8 mirrored products q_j*p_m: swapping the operand roles only
// permutes the products inside an instruction, whose sum is order-invariant (measured: tests/diag_mma_symmetry.py),
// so S[j][m] == S[m][j] bit for bit, on one rank and across ranks.
template <int PREC>
__device__ __forceinline__ void store_kcat_row(uint16_t* row, long long Dp, int d, const uint4 (&pk)[3], bool side_b) {
  *reinterpret_cast<uint4*>(row + d) = pk[0];
  if (PREC == PREC_FP16X2) {
    *reinterpret_cast<uint4*>(row + Dp + 2 * d) = side_b ? pk[1] : pk[0];
    *reinterpret_cast<uint4*>(row + Dp + 2 * d + 8) = side_b ? pk[0] : pk[1];
  } else if (PREC == PREC_BF16X3) {
    *reinterpret_cast<uint4*>(row + Dp + d) = pk[1];
    *reinterpret_cast<uint4*>(row + 2 * Dp + 2 * d) = side_b ? pk[1] : pk[0];
    *reinterpret_cast<uint4*>(row + 2 * Dp + 2 * d + 8) = side_b ? pk[0] : pk[1];
    *reinterpret_cast<uint4*>(row + 4 * Dp + 2 * d) = side_b ? pk[2] : pk[0];
    *reinterpret_cast<uint4*>(row + 4 * Dp + 2 * d + 8) = side_b ? pk[0] : pk[2];
  }
}

// Row i's statistics before a similarity sweep accumulates into them (caffe_set of the stat blobs, .cu:230-236)
__device__ __forceinline__ void reset_row_stats(const RowArrays& ra, long long i) {
  ra.st_minw[i] = f2ord(FLT_MAX); ra.st_maxw[i] = f2ord(-FLT_MAX);
  ra.st_maxb[i] = f2ord(-FLT_MAX); ra.st_maxall[i] = f2ord(-FLT_MAX);
  ra.cnt_same[i] = 0;
}

// exp(s - max) with the row constant pre-multiplied, m2 = max * log2(e): one FFMA + one MUFU.EX2 (relative error ~ (2 + 1.44|x|)
// ulp: 3e-7 for the |x| <= 2 of unit-norm embeddings).  Cheap enough to evaluate for EVERY pair, which keeps the row pass and the
// weight builder branch-free (the reference's expf, .cu:131, under a selection branch costs ~20 instructions per divergent hit).
// The same exponential is used forward and backward, so W = e / A stays consistent.
__device__ __forceinline__ float fast_exp_m2(float sv, float m2) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(fmaf(sv, LOG2E, -m2)));
  return y;
}

// --------------------------------------------------------------------------------------------
// absmax / asum  (caffe_gpu_asum .cu:400; operand pre-scale for PREC_FP16X2)
// --------------------------------------------------------------------------------------------
// x[4q .. 4q + 3]: one 16-byte load (VEC: x is 16-byte aligned) or four 4-byte loads
template <bool VEC>
__device__ __forceinline__ float4 load4(const float* __restrict__ x, long long q) {
  if (VEC) return __ldg(reinterpret_cast<const float4*>(x) + q);
  return make_float4(__ldg(x + 4 * q), __ldg(x + 4 * q + 1), __ldg(x + 4 * q + 2), __ldg(x + 4 * q + 3));
}
// This thread's share of sum |x| (and of max |x| when want_max) over x[0, n): groups of 4 a grid stride apart, four groups in flight,
// then the last n % 4 elements.  VEC: 16-byte loads (x 16-byte aligned); otherwise the same elements in the same order through
// 4-byte loads, so the asum top does not depend on where the caller's buffer starts.
template <bool VEC>
__device__ __forceinline__ void abs_sum_max(const float* __restrict__ x, long long n, long long t0, long long stride, bool want_max,
                                            float& sum, float& mx) {
  const long long n4 = n >> 2;
  long long i = t0;
  for (; i + 3 * stride < n4; i += 4 * stride) {
    const float4 a = load4<VEC>(x, i), b = load4<VEC>(x, i + stride), c = load4<VEC>(x, i + 2 * stride), d = load4<VEC>(x, i + 3 * stride);
    const float a0 = fabsf(a.x), a1 = fabsf(a.y), a2 = fabsf(a.z), a3 = fabsf(a.w), b0 = fabsf(b.x), b1 = fabsf(b.y), b2 = fabsf(b.z), b3 = fabsf(b.w);
    const float c0 = fabsf(c.x), c1 = fabsf(c.y), c2 = fabsf(c.z), c3 = fabsf(c.w), d0 = fabsf(d.x), d1 = fabsf(d.y), d2 = fabsf(d.z), d3 = fabsf(d.w);
    sum += (a0 + a1) + (a2 + a3) + (b0 + b1) + (b2 + b3) + (c0 + c1) + (c2 + c3) + (d0 + d1) + (d2 + d3);
    if (want_max) {
      mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(a0, a1), fmaxf(a2, a3)), fmaxf(fmaxf(b0, b1), fmaxf(b2, b3))));
      mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(c0, c1), fmaxf(c2, c3)), fmaxf(fmaxf(d0, d1), fmaxf(d2, d3))));
    }
  }
  for (; i < n4; i += stride) {
    const float4 a = load4<VEC>(x, i);
    sum += (fabsf(a.x) + fabsf(a.y)) + (fabsf(a.z) + fabsf(a.w));
    if (want_max) mx = fmaxf(mx, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))));
  }
  for (long long j = (n4 << 2) + t0; j < n; j += stride) { sum += fabsf(x[j]); if (want_max) mx = fmaxf(mx, fabsf(x[j])); }
}
// One kernel: per-block partial |x| sums (local rows) and max|x| (all rows), the reset of the per-row statistics, and --
// in the last block to finish (ticket) -- the final asum, the power-of-two operand scale and the reset of the step state.
// Returns true in the block that finished last (it has written the step's scalars to *bs).
__device__ __forceinline__ bool prep_reduce_body(const float* __restrict__ xl, long long nl, const float* __restrict__ xt, long long ntot,
                                                 float* __restrict__ partial, int want_scale, RowArrays ra, int Q, BlockScalars* bs) {
  __shared__ float s_sum[8], s_max[8];
  __shared__ int s_last;
  float sum = 0.f, mx = 0.f;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  // 16-byte loads, four in flight per thread (cudaMalloc'd / framework blobs are 16-byte aligned; otherwise 4-byte loads)
  const bool same_range = want_scale && xl == xt && nl == ntot;    // world == 1: one sweep gives both the sum and the maximum
  if ((reinterpret_cast<uintptr_t>(xl) & 15) == 0) abs_sum_max<true>(xl, nl, t0, stride, same_range, sum, mx);
  else abs_sum_max<false>(xl, nl, t0, stride, same_range, sum, mx);
  if (want_scale && !same_range) {
    if ((reinterpret_cast<uintptr_t>(xt) & 15) == 0) {
      const float4* x4 = reinterpret_cast<const float4*>(xt);
      const long long n4 = ntot >> 2;
      long long i = t0;
      for (; i + 3 * stride < n4; i += 4 * stride) {
        const float4 a = __ldg(x4 + i), b = __ldg(x4 + i + stride), c = __ldg(x4 + i + 2 * stride), d = __ldg(x4 + i + 3 * stride);
        mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))), fmaxf(fmaxf(fabsf(b.x), fabsf(b.y)), fmaxf(fabsf(b.z), fabsf(b.w)))));
        mx = fmaxf(mx, fmaxf(fmaxf(fmaxf(fabsf(c.x), fabsf(c.y)), fmaxf(fabsf(c.z), fabsf(c.w))), fmaxf(fmaxf(fabsf(d.x), fabsf(d.y)), fmaxf(fabsf(d.z), fabsf(d.w)))));
      }
      for (; i < n4; i += stride) { const float4 a = __ldg(x4 + i); mx = fmaxf(mx, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w)))); }
      for (long long j = (n4 << 2) + t0; j < ntot; j += stride) mx = fmaxf(mx, fabsf(xt[j]));
    } else {
      for (long long i = t0; i < ntot; i += stride) mx = fmaxf(mx, fabsf(xt[i]));
    }
  }
  for (long long i = t0; i < Q; i += stride) reset_row_stats(ra, i);
  sum = warp_sum(sum); mx = warp_max(mx);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_sum[w] = sum; s_max[w] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    sum = 0.f; mx = 0.f;
    for (int k = 0; k < (blockDim.x >> 5); ++k) { sum += s_sum[k]; mx = fmaxf(mx, s_max[k]); }
    partial[blockIdx.x] = sum; partial[1024 + blockIdx.x] = mx;
    __threadfence();
    s_last = (atomicAdd(&bs->ticket0, 1u) == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return false;
  __threadfence();
  __shared__ double s_dsum[8];
  double dsum = 0.0; mx = 0.f;
  for (int b = threadIdx.x; b < static_cast<int>(gridDim.x); b += blockDim.x) { dsum += __ldcg(&partial[b]); mx = fmaxf(mx, __ldcg(&partial[1024 + b])); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { dsum += __shfl_xor_sync(0xffffffffu, dsum, o); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
  if (l == 0) { s_dsum[w] = dsum; s_max[w] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    dsum = 0.0; mx = 0.f;
    for (int k = 0; k < (blockDim.x >> 5); ++k) { dsum += s_dsum[k]; mx = fmaxf(mx, s_max[k]); }
    bs->asum = static_cast<float>(dsum);
    bs->x_absmax = mx;
    float sc = 1.f, inv = 1.f;
    if (want_scale) { const PreScale ps = pre_scale(mx); sc = ps.scale; inv = ps.inv; }
    bs->x_scale = sc; bs->x_inv_scale = inv;
    bs->err = 0; bs->ticket = 0; bs->ticket2 = 0; bs->ticket0 = 0; bs->ticket3 = 0; bs->sel_active[0] = 0; bs->sel_active[1] = 0;
    bs->cand_n[0] = 0; bs->cand_n[1] = 0;
    bs->n_same = 0; bs->n_diff = 0;
  }
  return true;
}
__global__ void __launch_bounds__(256) prep_reduce_kernel(const float* __restrict__ xl, long long nl, const float* __restrict__ xt, long long ntot,
                                                          float* __restrict__ partial, int want_scale, RowArrays ra, int Q, BlockScalars* bs) {
  prep_reduce_body(xl, nl, xt, ntot, partial, want_scale, ra, Q, bs);
}
void launch_prep_reduce(const float* x_local, long long n_local, const float* x_total, long long n_total, float* partial,
                        int want_scale, RowArrays ra, int Q, BlockScalars* bs, cudaStream_t st) {
  long long nmax = n_local > n_total ? n_local : n_total;
  int nb = static_cast<int>((nmax + 256 * 16 - 1) / (256 * 16));
  if (nb < 1) nb = 1; if (nb > 592) nb = 592;
  prep_reduce_kernel<<<nb, 256, 0, st>>>(x_local, n_local, x_total, n_total, partial, want_scale, ra, Q, bs);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// operand split: x_total fp32 [N x D] -> Xs[s][N][ldXs] (K-major for the similarity GEMM) and the transposed
// XsT[s][D][ldXsT] (K-major for the gradient GEMM whose K is the sample index); XlT = local columns only.
// --------------------------------------------------------------------------------------------
// Block = 256 threads, tile = 32 rows (n) x 64 features (d).  Thread (nl = t/8, dg = t%8) converts 8 consecutive features of
// one row: two 16-byte loads, one 16-byte store per piece / section; the transposed pieces go through a shared tile so
// that they, too, are written as 16-byte row segments.
struct SplitArgs {
  const float* x; int N, D;
  uint16_t* Xs; long long ldXs; uint16_t* XsT; long long ldXsT; uint16_t* XlT; long long ldXlT; int row0, Q;
  uint16_t *XcatA, *XcatB; long long Dp;
};
// The 8 features thread t of a block converts in tile (tile_d, tile_n): two 16-byte loads (issued early by the fused kernel).
__device__ __forceinline__ void split_load(const SplitArgs& a, int tile_d, int tile_n, float (&v)[8]) {
  const float* __restrict__ x = a.x; const int N = a.N, D = a.D;
  const int t = threadIdx.x, nl = t >> 3, dg = t & 7;
  const int n = tile_n * 32 + nl, d = tile_d * 64 + 8 * dg;
  const bool rowok = n < N;
  if (rowok && d + 7 < D && (D & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {   // 16-byte loads need an aligned base
    const float4 a4 = *reinterpret_cast<const float4*>(x + static_cast<long long>(n) * D + d);
    const float4 b4 = *reinterpret_cast<const float4*>(x + static_cast<long long>(n) * D + d + 4);
    v[0] = a4.x; v[1] = a4.y; v[2] = a4.z; v[3] = a4.w; v[4] = b4.x; v[5] = b4.y; v[6] = b4.z; v[7] = b4.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = (rowok && d + e < D) ? x[static_cast<long long>(n) * D + d + e] : 0.f;
  }
}
// One 32-row x 64-feature tile (tile_n, tile_d) by one block of 256 threads from the values split_load fetched.  `buf` alternates
// between consecutive tiles of a block: the transposition tile is double-buffered, so ONE barrier per tile is enough.
template <int PREC>
__device__ __forceinline__ void split_tile(const SplitArgs& a, float sc, int tile_d, int tile_n, const float (&v)[8], int buf) {
  const int N = a.N, D = a.D;
  uint16_t* __restrict__ Xs = a.Xs; const long long ldXs = a.ldXs; uint16_t* __restrict__ XsT = a.XsT; const long long ldXsT = a.ldXsT;
  uint16_t* __restrict__ XlT = a.XlT; const long long ldXlT = a.ldXlT; const int row0 = a.row0, Q = a.Q;
  uint16_t* __restrict__ XcatA = a.XcatA; uint16_t* __restrict__ XcatB = a.XcatB; const long long Dp = a.Dp;
  constexpr int NS = SPLIT_FORMATS[PREC].pieces;
  __shared__ __align__(16) uint16_t tile2[2][NS][64][40];  // [buffer][piece][d][n], row padded to 80 bytes (16-byte aligned, spreads banks)
  uint16_t (*tile)[64][40] = tile2[buf];
  const int n0 = tile_n * 32, d0 = tile_d * 64;
  const int t = threadIdx.x, nl = t >> 3, dg = t & 7;
  const int n = n0 + nl, d = d0 + 8 * dg;
  uint16_t p[8][3];
  uint4 pk[3];
  const bool rowok = n < N;
  split8<PREC>(v, sc, p, pk);
#pragma unroll
  for (int s = 0; s < NS; ++s)
#pragma unroll
    for (int e = 0; e < 8; ++e) tile[s][8 * dg + e][nl] = p[e][s];
  // every destination row is padded to a multiple of 64 elements (Dp), so whole 16-byte groups can be stored even when
  // D is ragged: the excess elements are zeros (v = 0 above), which is what the similarity GEMM reads past D (its K extent is Dp
  // per segment) and which lies beyond the TMA extent of every other map
  if (rowok && d < Dp) {
    const long long ps = static_cast<long long>(N) * ldXs;
    if (Xs)      // NULL when the similarity GEMM reads the K-concatenated operands below
#pragma unroll
      for (int s = 0; s < NS; ++s) *reinterpret_cast<uint4*>(Xs + s * ps + static_cast<long long>(n) * ldXs + d) = pk[s];
    // K-concatenated operands of the bitwise-symmetric similarity GEMM: every row in the B format, and the rank's own rows, the only
    // ones that are ever an A operand, also in the A format
    if (PREC != PREC_BF16 && XcatA) {
      const long long kcat = mma_passes(NS) * Dp;
      store_kcat_row<PREC>(XcatB + static_cast<long long>(n) * kcat, Dp, d, pk, true);
      if (n >= row0 && n < row0 + Q) store_kcat_row<PREC>(XcatA + static_cast<long long>(n) * kcat, Dp, d, pk, false);
    }
  }
  __syncthreads();
  // transposed pieces: thread (dl = t/4, nc = t%4) stores 8 consecutive rows n of feature d0 + dl
  const int dl = t >> 2, nc = t & 3;
  const int dd = d0 + dl, nn = n0 + 8 * nc;
  if (dd < D && nn < N) {
    const long long pt = static_cast<long long>(D) * ldXsT;
    const long long pl = static_cast<long long>(D) * ldXlT;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const uint4 q = *reinterpret_cast<const uint4*>(&tile[s][dl][8 * nc]);
      *reinterpret_cast<uint4*>(XsT + s * pt + static_cast<long long>(dd) * ldXsT + nn) = q;     // ldXsT, nn multiples of 8
      if (XlT && nn >= row0 && nn < row0 + Q) {
        if (((nn - row0) & 7) == 0 && nn + 8 <= row0 + Q) *reinterpret_cast<uint4*>(XlT + s * pl + static_cast<long long>(dd) * ldXlT + (nn - row0)) = q;
        else
          for (int e = 0; e < 8; ++e)
            if (nn + e < row0 + Q && nn + e < N) XlT[s * pl + static_cast<long long>(dd) * ldXlT + (nn + e - row0)] = tile[s][dl][8 * nc + e];
      } else if (XlT && nn < row0 && nn + 8 > row0) {
        for (int e = 0; e < 8; ++e)
          if (nn + e >= row0 && nn + e < row0 + Q && nn + e < N) XlT[s * pl + static_cast<long long>(dd) * ldXlT + (nn + e - row0)] = tile[s][dl][8 * nc + e];
      }
    }
  }
}
template <int PREC>
__global__ void __launch_bounds__(256) split_kernel(SplitArgs a, const BlockScalars* __restrict__ bs) {
  float v[8];
  split_load(a, blockIdx.x, blockIdx.y, v);
  split_tile<PREC>(a, (PREC == PREC_FP16X2) ? bs->x_scale : 1.f, blockIdx.x, blockIdx.y, v, 0);
}
void launch_split(const float* x_total, int N, int D, int prec, const BlockScalars* bs, uint16_t* Xs, long long ldXs,
                  uint16_t* XsT, long long ldXsT, uint16_t* XlT, long long ldXlT, int row0_local, int Q,
                  uint16_t* XcatA, uint16_t* XcatB, long long Dp, cudaStream_t st) {
  dim3 grid((D + 63) / 64, (N + 31) / 32);
  const SplitArgs a{x_total, N, D, Xs, ldXs, XsT, ldXsT, XlT, ldXlT, row0_local, Q, XcatA, XcatB, Dp};
  with_prec(prec, [&](auto P) { split_kernel<P><<<grid, 256, 0, st>>>(a, bs); });
  count_launch();
}

// --------------------------------------------------------------------------------------------
// statistics init / reference row statistics (caffe_set of the three stat blobs, .cu:230-236)
// --------------------------------------------------------------------------------------------
// One block per row; same outputs as the sim-GEMM epilogue.  Used by the SIMT cross-check backend and by tests.
__global__ void row_stats_ref_kernel(const __grid_constant__ SimRows sim, RowArrays ra) {
  const int i = sim.row0 + blockIdx.x;
  const float li = __ldg(sim.lab_rows + i);
  float minw = FLT_MAX, maxw = -FLT_MAX, maxb = -FLT_MAX, maxall = -FLT_MAX;
  int cnt = 0;
  const float* row = sim.row(i);
  for (int j = threadIdx.x; j < sim.N; j += blockDim.x) {
    if (j == sim.self_col(i)) continue;
    const float v = __ldg(row + j);
    maxall = fmaxf(maxall, v);
    if (__ldg(sim.lab_cols + j) == li) { minw = fminf(minw, v); maxw = fmaxf(maxw, v); ++cnt; } else maxb = fmaxf(maxb, v);
  }
  minw = warp_min(minw); maxw = warp_max(maxw); maxb = warp_max(maxb); maxall = warp_max(maxall); cnt = warp_sum_i(cnt);
  if ((threadIdx.x & 31) == 0) {
    atomicMin(&ra.st_minw[i], f2ord(minw)); atomicMax(&ra.st_maxw[i], f2ord(maxw));
    atomicMax(&ra.st_maxb[i], f2ord(maxb)); atomicMax(&ra.st_maxall[i], f2ord(maxall));
    if (cnt) atomicAdd(&ra.cnt_same[i], cnt);
  }
}
void launch_row_stats_ref(SimRows sim, RowArrays ra, cudaStream_t st) {
  row_stats_ref_kernel<<<sim.rows, 256, 0, st>>>(sim, ra);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// thresholds (.cu:275-337): thresholds_one_block (thresholds.cuh).  Non-relative modes and the pos==size-1 relative shortcut are
// closed forms of the row statistics; general relative modes arm the radix selects below.
// --------------------------------------------------------------------------------------------
// SIMT backend (the tensor-core similarity sweep runs the pick in its last CTA)
__global__ void __launch_bounds__(1024) thresholds_kernel(RowArrays ra, int Q, int N, MiningParams mp, BlockScalars* bs) {
  __shared__ __align__(8) unsigned char scratch[THRESHOLDS_SCRATCH_BYTES];
  thresholds_one_block(ra, Q, N, mp, bs, scratch, nullptr);
}
// world scope (npair_config.global_scope): every rank reduces the world's block statistics in the same order -> identical thresholds
__global__ void thresholds_world_kernel(const BlockStats* __restrict__ xall, int xstride, int world, long long N, MiningParams mp,
                                        BlockScalars* bs) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  finish_thresholds(xall, world, xstride, static_cast<unsigned long long>(N), N, mp, bs);
}
void launch_thresholds_world(const float* xall, int xstride, int world, long long N, MiningParams mp, BlockScalars* bs, cudaStream_t st) {
  thresholds_world_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const BlockStats*>(xall), xstride, world, N, mp, bs);
  count_launch();
}
void launch_thresholds(RowArrays ra, int Q, int N, MiningParams mp, BlockScalars* bs, cudaStream_t st) {
  thresholds_kernel<<<1, 1024, 0, st>>>(ra, Q, N, mp, bs);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// Relative thresholds = order statistics of the masked similarities (replaces the unconditional std::sorts of .cu:266-273
// and the list indexing of .cu:282-290, :300-304, :313-321, :331-335).  MSB-first radix select on the order-preserving
// uint32 keys, digits of 11 / 11 / 10 bits.  Similarities of one row are clustered (a few binades), so the first digit
// already narrows the k-th element down to a few percent of the row: those CANDIDATES are compacted (21-bit remainders) and the
// last two digits are decided on the compact list -- S is read once from HBM (LOCAL: one more time from L1/L2; GLOBAL: twice).
// Both sides (same-label list for AP, diff-label list for AN) are handled in the same sweep when both are relative.
// The self pair is in neither list, whatever its label (.cu:54): it is recognised by its column, never by its label, since a NaN
// label is not equal to itself.
// --------------------------------------------------------------------------------------------
#define NPAIR_SEL_BINS 2048

// Histogram increment as ONE shared-memory reduction per lane.  A plain atomicAdd(&hist[d], 1) is rewritten by the compiler into a
// loop over the warp's distinct addresses (leader election + ATOMS.POPC.INC per address): ~20 instructions per distinct bin, the
// bulk of the select kernels' instruction count in the first round-2 version.  The hardware resolves same-address conflicts itself.
__device__ __forceinline__ void smem_inc(unsigned int* p) {
  asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(p))) : "memory");
}
__device__ __forceinline__ void smem_inc_off(unsigned int* base, uint32_t byte_off) {
  asm volatile("red.shared.add.u32 [%0], 1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(base)) + byte_off) : "memory");
}
__device__ __forceinline__ void smem_dec(unsigned int* p) {
  asm volatile("red.shared.add.u32 [%0], -1;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(p))) : "memory");
}

// ---- parts shared by the select kernels ----
#define NPAIR_LSEL_SCAP 128                // same-label entries kept per row (LOCAL)

// Value order -> raw digit of the top `bits` bits of a float (sign first): orders [0, 2^(bits-1)) are the negative floats, whose raw
// digits descend
__device__ __forceinline__ uint32_t raw_digit_of_order(uint32_t o, int bits) {
  const uint32_t half = 1u << (bits - 1);
  return o < half ? 2u * half - 1u - o : o - half;
}
// Below a top digit of the raw bits, the remainders of negative floats sort descending: XOR with this mask (the low rem_bits when the
// sign bit of `bits` is set) puts a remainder in value order, and back again
__device__ __forceinline__ uint32_t rem_flip(uint32_t bits, int rem_bits) { return (bits >> 31) ? (1u << rem_bits) - 1u : 0u; }

template <class T>
__device__ __forceinline__ T warp_incl_sum(T x, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += t; }
  return x;
}

// Bin of 0-based rank r among bins 0 .. nb-1 taken in index order, bin b holding cnt(b) entries (cnt folds in any bin-index map); by a
// warp, nb a multiple of 32 and at most 1024.  Lane l sums bins [l * nb/32, (l+1) * nb/32); the winning lane's bins are then scanned
// one per lane.  Returns the bin and *r_in, the rank inside it (warp-uniform); nb when r is out of range.
template <class C>
__device__ __forceinline__ int warp_find_bin(C cnt, int nb, unsigned int r, unsigned int* r_in, int lane) {
  const int per = nb >> 5;
  unsigned int mine = 0;
  for (int b = 0; b < per; ++b) mine += cnt(lane * per + b);
  const unsigned int before = warp_incl_sum(mine, lane) - mine;
  const unsigned int hit = __ballot_sync(0xffffffffu, mine && r >= before && r < before + mine);
  if (!hit) return nb;
  const int src = __ffs(hit) - 1;
  const unsigned int base = __shfl_sync(0xffffffffu, before, src);
  const int bin = src * per + lane;
  const unsigned int h = lane < per ? cnt(bin) : 0u;
  const unsigned int bef = base + warp_incl_sum(h, lane) - h;
  const int src2 = __ffs(__ballot_sync(0xffffffffu, h && r >= bef && r < bef + h)) - 1;
  *r_in = r - __shfl_sync(0xffffffffu, bef, src2);
  return __shfl_sync(0xffffffffu, bin, src2);
}

// A same-label entry (raw bits) joins its row's list; past NPAIR_LSEL_SCAP entries it is only counted, and the row's sides that need
// the list take the slow path
__device__ __forceinline__ void same_append(unsigned int* n, uint32_t* list, uint32_t bits) {
  const unsigned int k = atomicAdd(n, 1u);
  if (k < NPAIR_LSEL_SCAP) list[k] = bits;
}

// Of the n ordered keys key(0 .. n-1), the one of 0-based rank pos (ties by index) is stored to *out as a threshold, by the thread that
// holds it: threads e0, e0 + step, ... take one key each and count the keys before it
template <class K>
__device__ __forceinline__ void store_key_of_rank(K key, unsigned int n, unsigned int pos, unsigned int e0, unsigned int step, float* out) {
  for (unsigned int e = e0; e < n; e += step) {
    const uint32_t ke = key(e);
    unsigned int rk = 0;
    for (unsigned int t = 0; t < n; ++t) { const uint32_t kt = key(t); rk += (kt < ke || (kt == ke && t < e)) ? 1u : 0u; }
    if (rk == pos) *out = clamp_thr(ord2f(ke));
  }
}

// ---- LOCAL: ONE WARP per row, warp-private histogram -- no block barriers, no block-wide scans ----
// sweep 1  digit 1 (top 10 bits of the RAW float bits: 3 instructions per element, no label branch) of every column into the warp's
//          histogram; the few same-label entries (and the self pair) are kept in a small list on the side
// pick     the excluded keys (same-label entries, self pair) are taken out of the histogram again; bins are walked in value order
//          (negative floats: descending raw digit) to find the bin of the wanted rank
// sweep 2  (L1 / L2) elements of that bin -> per-LANE private candidate lists in shared memory (two predicated instructions per
//          match: no ballots, no atomics); 22-bit remainders
// tail     three more digits (8 + 7 + 7 bits) over the candidate lists, excluded keys subtracted per digit
// Anything that does not fit the fast path (more than 128 same-label entries, a lane with more than 48 candidates) is redone
// by slow_select_row: plain sweeps of the row, one digit per sweep, label test per element.
#define NPAIR_LSEL_WARPS 8
#define NPAIR_LSEL_D1 1024                 // bins of the first digit
#define NPAIR_LSEL_LCAP 48                 // candidates per lane
#define NPAIR_LSEL_U 4                     // 16-byte loads in flight per lane and array
struct LselWarp {
  unsigned int hist[NPAIR_LSEL_D1];
  uint32_t cand[32 * NPAIR_LSEL_LCAP];     // [slot][lane]: lane-private lists, bank = lane
  uint32_t same[NPAIR_LSEL_SCAP];          // raw bits of the same-label entries (self pair excluded)
  unsigned int n_same, pad_[3];            // keeps sizeof a multiple of 16 (16-byte stores into hist)
};
static_assert(sizeof(LselWarp) % 16 == 0, "LselWarp must keep 16-byte alignment in an array");

// Generic (slow) select of one side of one row by a warp: 32-bit ordered keys, digits of 10/10/10/2 bits, one sweep of the row per digit.
__device__ __noinline__ uint32_t slow_select_row(const float* __restrict__ row, int N, const float* __restrict__ lab_cols, float li, int self_col,
                                                 int side, unsigned int rank, unsigned int* hist /*[1024]*/, int lane) {
  uint32_t prefix = 0, mask = 0;
  int shift = 22;
  for (int pass = 0; pass < 4; ++pass) {
    const int bits = pass < 3 ? 10 : 2;
    if (pass == 3) shift = 0;
    const int nb = 1 << bits;
    for (int b = lane; b < 1024; b += 32) hist[b] = 0;
    __syncwarp();
    for (int j = lane; j < N; j += 32) {
      if (j == self_col) continue;
      if ((lab_cols[j] == li) != (side == 0)) continue;
      const uint32_t key = f2ord(row[j]);
      if ((key & mask) == prefix) smem_inc(&hist[(key >> shift) & (nb - 1)]);
    }
    __syncwarp();
    unsigned int r2;
    const int d = warp_find_bin([&](int b) { return hist[b]; }, nb < 32 ? 32 : nb, rank, &r2, lane);
    prefix |= static_cast<uint32_t>(d) << shift; mask |= static_cast<uint32_t>(nb - 1) << shift; rank = r2;
    shift -= 10;
    __syncwarp();
  }
  return prefix;
}

__global__ void __launch_bounds__(32 * NPAIR_LSEL_WARPS, 2) local_select_kernel(const __grid_constant__ SimRows sim, int side_mask /*1 AP, 2 AN*/, float sn_ap,
                                                                              float sn_an, RowArrays ra, BlockScalars* bs) {
  extern __shared__ __align__(16) unsigned char lsel_smem[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  LselWarp& W = reinterpret_cast<LselWarp*>(lsel_smem)[w];
  const bool want_same = side_mask & 1, want_diff = side_mask & 2;
  const int N = sim.N;
  const float* lab_cols = sim.lab_cols;
  const bool lab_aligned = (reinterpret_cast<uintptr_t>(lab_cols) & 15) == 0;
  const int nwarps = gridDim.x * NPAIR_LSEL_WARPS;
  for (int i = sim.row0 + blockIdx.x * NPAIR_LSEL_WARPS + w; i < sim.row0 + sim.rows; i += nwarps) {
    const float li = __ldg(sim.lab_rows + i);
    const int self_col = sim.self_col(i);
    const float* row = sim.row(i);
    const int cs = ra.cnt_same[i];
    // ---------------- sweep 1 ----------------
    for (int b = lane * 4; b < NPAIR_LSEL_D1; b += 128) *reinterpret_cast<uint4*>(&W.hist[b]) = make_uint4(0u, 0u, 0u, 0u);
    if (lane == 0) W.n_same = 0;
    __syncwarp();
    const int n_vec = lab_aligned ? (N & ~127) : 0;               // whole 128-column groups with aligned labels: 16-byte loads
    for (int j4 = lane * 4; j4 < n_vec; j4 += 128 * NPAIR_LSEL_U) {   // NPAIR_LSEL_U groups (16-byte loads of S and of the labels) in flight per lane
      uint4 v[NPAIR_LSEL_U]; float4 l[NPAIR_LSEL_U];
#pragma unroll
      for (int u = 0; u < NPAIR_LSEL_U; ++u) {
        const int jj = j4 + 128 * u;
        if (jj < n_vec) { v[u] = __ldg(reinterpret_cast<const uint4*>(row + jj)); l[u] = __ldg(reinterpret_cast<const float4*>(lab_cols + jj)); }
      }
#pragma unroll
      for (int u = 0; u < NPAIR_LSEL_U; ++u) {
        const int jj = j4 + 128 * u;
        if (jj >= n_vec) continue;
        const uint32_t vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
        const float ll[4] = {l[u].x, l[u].y, l[u].z, l[u].w};
        if (want_diff) {
#pragma unroll
          for (int c = 0; c < 4; ++c) smem_inc_off(W.hist, (vv[c] >> 20) & 0xFFCu);
        }
        if (ll[0] == li || ll[1] == li || ll[2] == li || ll[3] == li) {
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (ll[c] == li && jj + c != self_col) same_append(&W.n_same, W.same, vv[c]);
        }
      }
    }
    for (int j = n_vec + lane; j < N; j += 32) {                  // ragged tail / unaligned labels
      const uint32_t b = __float_as_uint(row[j]);
      if (want_diff) smem_inc(&W.hist[b >> 22]);
      if (lab_cols[j] == li && j != self_col) same_append(&W.n_same, W.same, b);
    }
    __syncwarp();
    const unsigned int ns = W.n_same;                             // == cs
    const uint32_t self_bits = __float_as_uint(row[self_col]);
    // ---------------- AP side: the same-label list is short ----------------
    if (want_same) {
      unsigned long long pos = 0;
      if (cs == 0) { if (lane == 0) { atomicOr(&bs->err, DERR_EMPTY_LIST); ra.posi_thr[i] = 0.f; } }
      else if (!pos_index(sn_ap, static_cast<unsigned long long>(cs), pos)) { if (lane == 0) { atomicOr(&bs->err, DERR_POS_RANGE); ra.posi_thr[i] = 0.f; } }
      else if (ns <= 32) {                                        // rank by counting inside the warp
        store_key_of_rank([&](unsigned int t) { return f2ord(__uint_as_float(W.same[t])); }, ns, static_cast<unsigned int>(pos), lane, 32,
                          &ra.posi_thr[i]);                                                                // .cu:288
      } else {
        const float thr = clamp_thr(ord2f(slow_select_row(row, N, lab_cols, li, self_col, 0, static_cast<unsigned int>(pos), W.hist + 0, lane)));
        if (lane == 0) ra.posi_thr[i] = thr;
        // the slow path used the histogram: rebuild digit 1 for the diff side below by falling into its slow path as well
        if (want_diff && lane == 0) W.n_same = NPAIR_LSEL_SCAP + 1;
      }
      __syncwarp();
    }
    // ---------------- AN side ----------------
    if (want_diff) {
      unsigned long long pos = 0;
      float thr = 0.f;
      const unsigned long long size = static_cast<unsigned long long>(N - 1 - cs);
      if (size == 0) { if (lane == 0) atomicOr(&bs->err, DERR_EMPTY_LIST); }
      else if (!pos_index(sn_an, size, pos)) { if (lane == 0) atomicOr(&bs->err, DERR_POS_RANGE); }
      else if (W.n_same > NPAIR_LSEL_SCAP) {
        thr = clamp_thr(ord2f(slow_select_row(row, N, lab_cols, li, self_col, 1, static_cast<unsigned int>(pos), W.hist, lane)));
      } else {
        // excluded keys (same-label entries + the self pair) leave the histogram; then walk the bins in value order
        for (unsigned int e = lane; e <= ns; e += 32) smem_dec(&W.hist[(e < ns ? W.same[e] : self_bits) >> 22]);
        __syncwarp();
        // the raw bins are read in value order; the bin exists: pos < size = sum of the bins
        unsigned int rank;
        const uint32_t raw = raw_digit_of_order(static_cast<uint32_t>(warp_find_bin([&](int o) { return W.hist[raw_digit_of_order(o, 10)]; },
                                                                                    NPAIR_LSEL_D1, static_cast<unsigned int>(pos), &rank, lane)), 10);
        // ---------------- sweep 2: that bin's elements -> lane-private candidate lists ----------------
        unsigned int cnt = 0;
        for (int j4 = lane * 4; j4 < n_vec; j4 += 128 * NPAIR_LSEL_U) {
          uint4 v[NPAIR_LSEL_U];
#pragma unroll
          for (int u = 0; u < NPAIR_LSEL_U; ++u) if (j4 + 128 * u < n_vec) v[u] = __ldg(reinterpret_cast<const uint4*>(row + j4 + 128 * u));
#pragma unroll
          for (int u = 0; u < NPAIR_LSEL_U; ++u) {
            if (j4 + 128 * u >= n_vec) continue;
            const uint32_t vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
            for (int c = 0; c < 4; ++c)
              if ((vv[c] >> 22) == raw) { if (cnt < NPAIR_LSEL_LCAP) W.cand[cnt * 32 + lane] = vv[c] & 0x3FFFFFu; ++cnt; }
          }
        }
        for (int j = n_vec + lane; j < N; j += 32) {
          const uint32_t b = __float_as_uint(row[j]);
          if ((b >> 22) == raw) { if (cnt < NPAIR_LSEL_LCAP) W.cand[cnt * 32 + lane] = b & 0x3FFFFFu; ++cnt; }
        }
        if (__any_sync(0xffffffffu, cnt > NPAIR_LSEL_LCAP)) {
          thr = clamp_thr(ord2f(slow_select_row(row, N, lab_cols, li, self_col, 1, static_cast<unsigned int>(pos), W.hist, lane)));
        } else {
          // ---------------- tail: 8 + 7 + 7 bits over the candidates; excluded keys of this bin are subtracted per digit ----------------
          const uint32_t flip = rem_flip(raw << 22, 22);
          uint32_t pre = 0, msk = 0;
          const int shifts[3] = {14, 7, 0}, nbits[3] = {8, 7, 7};
#pragma unroll
          for (int ps = 0; ps < 3; ++ps) {
            const int nb = 1 << nbits[ps];
            for (int b = lane * 4; b < nb; b += 128) *reinterpret_cast<uint4*>(&W.hist[b]) = make_uint4(0u, 0u, 0u, 0u);
            __syncwarp();
            for (unsigned int e = 0; e < cnt; ++e) {
              const uint32_t k = W.cand[e * 32 + lane] ^ flip;
              if ((k & msk) == pre) smem_inc(&W.hist[(k >> shifts[ps]) & (nb - 1)]);
            }
            __syncwarp();
            for (unsigned int e = lane; e <= ns; e += 32) {
              const uint32_t b = e < ns ? W.same[e] : self_bits;
              const uint32_t k = (b & 0x3FFFFFu) ^ flip;
              if ((b >> 22) == raw && (k & msk) == pre) smem_dec(&W.hist[(k >> shifts[ps]) & (nb - 1)]);
            }
            __syncwarp();
            unsigned int r2;
            const int d = warp_find_bin([&](int b) { return W.hist[b]; }, nb, rank, &r2, lane);
            pre |= static_cast<uint32_t>(d & (nb - 1)) << shifts[ps]; msk |= static_cast<uint32_t>(nb - 1) << shifts[ps]; rank = r2;
            __syncwarp();
          }
          thr = clamp_thr(__uint_as_float((raw << 22) | (pre ^ flip)));
        }
      }
      if (lane == 0) ra.nega_thr[i] = thr;                        // .cu:319
      __syncwarp();
    }
  }
}

// ---- LOCAL, rows of up to 8192 columns: ONE BLOCK per row, the row stays in registers ----
// The warp-per-row kernel above is bound by its instruction count and by its few warps in flight (ncu: 56 M warp instructions, 29 %
// issue slots with 16 warps per SM).  This kernel holds a row in the registers of 256 threads (8 independent 16-byte loads each, S is
// read ONCE) and bins by VALUE with three instructions per entry:
//   pass 0   label test: entries with the row's label go to the short same-label list, and they and the self pair (by column: a
//            NaN-labelled row's self pair has no label match) are replaced by NaN in the registers -- fminf / fmaxf skip NaN, so the
//            value range [lo, hi] of the entries that stay needs no branch
//   pass 1   bin*4 = mantissa of fmaf(s, 4*2048/(hi-lo), 2^23 + 4 - lo*that): one FFMA, one AND, one shared-memory reduction.  The map
//            is monotone in s, so the wanted rank lies in the bin where the running count crosses it; bins hold a few dozen entries and
//            lanes rarely collide.  NaN lands in bin 4095, which nobody reads.
//   pick     the bin's entries (same registers, same three instructions) -> ordered keys in shared memory, ranked by counting
//            (<= 256 of them).  A fuller bin (outliers stretching the range, masses of duplicates), or a range the float map cannot
//            resolve, is refined from the registers instead, 11 bits of the ORDERED KEY at a time.
// The next row's loads are issued as soon as the registers are free, before the pick.  (Measured: keeping TWO rows in registers, the
// next row's loads a whole iteration ahead at 2 blocks per SM, is slower: 153 against 140 us.)
#define NPAIR_LSB_THREADS 256
#define NPAIR_LSB_VPT 8                    // 16-byte groups per thread: 256 * 8 * 4 = 8192 columns
#define NPAIR_LSB_BINS 2048
#define NPAIR_LSB_HIST 2304                // bins the find walks: 1 + 2048 + slack (the value map is shifted up by one bin); multiple of 256
#define NPAIR_LSB_CCAP 256                 // bin population ranked by counting
#ifndef NPAIR_LSB_MINB
#define NPAIR_LSB_MINB 3                   // resident blocks per SM (80 registers)
#endif
struct LselBlock {
  unsigned int hist[4096];                 // [0, NPAIR_LSB_HIST) are cleared and read; 4095 collects the NaN (excluded) entries
  uint32_t cand[NPAIR_LSB_CCAP];
  uint32_t same[NPAIR_LSEL_SCAP];
  unsigned int n_same, n_cand;
  unsigned int warp_tot[NPAIR_LSB_THREADS / 32];
  unsigned int out[3];                     // find: {bin, rank inside the bin, population}
  float red_min[NPAIR_LSB_THREADS / 32], red_max[NPAIR_LSB_THREADS / 32];
  uint32_t red_klo[NPAIR_LSB_THREADS / 32], red_khi[NPAIR_LSB_THREADS / 32];
};

// Bin of 0-based rank r among hist[0 .. PER * 256) in index order, every thread holding PER consecutive bins in registers.  Two
// barriers; the result is in B.out afterwards (bin == PER * 256: rank out of range).
template <int PER>
__device__ __forceinline__ void block_find_bin_u32(LselBlock& B, unsigned int r) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  unsigned int h[PER], mine = 0;
#pragma unroll
  for (int q = 0; q < PER; ++q) { h[q] = B.hist[tid * PER + q]; mine += h[q]; }
  const unsigned int incl = warp_incl_sum(mine, lane);
  if (lane == 31) B.warp_tot[w] = incl;
  if (tid == 0) B.out[0] = static_cast<unsigned int>(PER * NPAIR_LSB_THREADS);
  __syncthreads();
  unsigned int before = incl - mine;
#pragma unroll
  for (int k = 0; k < NPAIR_LSB_THREADS / 32; ++k) before += (k < w) ? B.warp_tot[k] : 0u;
  if (mine && r >= before && r < before + mine) {                  // exactly one thread
    unsigned int cum = before;
    int b = 0;
#pragma unroll
    for (int q = 0; q < PER - 1; ++q) { if (b == q && cum + h[q] <= r) { cum += h[q]; b = q + 1; } }
    unsigned int hb = h[0];
#pragma unroll
    for (int q = 1; q < PER; ++q) hb = (b == q) ? h[q] : hb;
    B.out[0] = static_cast<unsigned int>(tid * PER + b); B.out[1] = r - cum; B.out[2] = hb;
  }
  __syncthreads();
}

__device__ __forceinline__ uint4 ldg_stream_u4(const float* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
// byte offset (bin * 4) of an entry in the histogram: monotone in f; NaN -> 0x3FFC
__device__ __forceinline__ uint32_t lsb_off(uint32_t bits, float s4, float c0) { return __float_as_uint(__fmaf_rn(__uint_as_float(bits), s4, c0)) & 0x3FFCu; }

__global__ void __launch_bounds__(NPAIR_LSB_THREADS, NPAIR_LSB_MINB) local_select_block_kernel(const __grid_constant__ SimRows sim, int side_mask /*1 AP, 2 AN*/,
                                                                                   float sn_ap, float sn_an, RowArrays ra, BlockScalars* bs) {
  __shared__ __align__(16) LselBlock B;
  constexpr uint32_t kNaN = 0x7FFFFFFFu;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const bool want_same = side_mask & 1, want_diff = side_mask & 2;
  // whole 4-column groups come through 16-byte loads (rows start 128-byte aligned: ldS is a multiple of 32); the last N % 4 columns
  // sit in one extra register of threads 0..2
  const int N = sim.N;
  const float* lab_cols = sim.lab_cols;
  const int n4 = N & ~3;
  const bool has_tail = tid < N - n4;
  uint32_t v[4 * NPAIR_LSB_VPT + 1];       // [32] = the tail column (NaN where there is none)
  const int row_end = sim.row0 + sim.rows;
  int i = sim.row0 + blockIdx.x;
  auto load_row = [&](int r) {
    const float* row = sim.row(r);
#pragma unroll
    for (int u = 0; u < NPAIR_LSB_VPT; ++u) {
      const int jj = (u * NPAIR_LSB_THREADS + tid) * 4;
      uint4 t = make_uint4(kNaN, kNaN, kNaN, kNaN);
      if (jj < n4) t = ldg_stream_u4(row + jj);
      v[4 * u] = t.x; v[4 * u + 1] = t.y; v[4 * u + 2] = t.z; v[4 * u + 3] = t.w;
    }
    v[4 * NPAIR_LSB_VPT] = has_tail ? __float_as_uint(row[n4 + tid]) : kNaN;
  };
  if (i < row_end) load_row(i);
  for (; i < row_end; i += gridDim.x) {
    const float li = __ldg(sim.lab_rows + i);
    const int self_col = sim.self_col(i);
    const int cs = ra.cnt_same[i];
    for (int b = tid * 4; b < NPAIR_LSB_HIST; b += NPAIR_LSB_THREADS * 4) *reinterpret_cast<uint4*>(&B.hist[b]) = make_uint4(0u, 0u, 0u, 0u);
    if (tid == 0) { B.n_same = 0; B.n_cand = 0; }
    __syncthreads();          // publishes the reset (the previous row's readers are behind the loop-end barrier)
    // ---------------- pass 0: labels -> same-label list, NaN in the registers; value range of the entries that stay ----------------
    float mn = FLT_MAX, mx = -FLT_MAX;
#pragma unroll
    for (int u = 0; u < NPAIR_LSB_VPT; ++u) {
      const int jj = (u * NPAIR_LSB_THREADS + tid) * 4;
      if (jj < n4) {
        const float4 l = __ldg(reinterpret_cast<const float4*>(lab_cols + jj));
        const float ll[4] = {l.x, l.y, l.z, l.w};
        if (sim.self_in4(i, jj) || l.x == li || l.y == li || l.z == li || l.w == li) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (ll[c] == li && jj + c != self_col) same_append(&B.n_same, B.same, v[4 * u + c]);
            if (ll[c] == li || jj + c == self_col) v[4 * u + c] = kNaN;
          }
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) { mn = fminf(mn, __uint_as_float(v[4 * u + c])); mx = fmaxf(mx, __uint_as_float(v[4 * u + c])); }
      }
    }
    if (has_tail) {
      const int j = n4 + tid;
      const bool same = lab_cols[j] == li;
      if (same && j != self_col) same_append(&B.n_same, B.same, v[4 * NPAIR_LSB_VPT]);
      if (same || j == self_col) v[4 * NPAIR_LSB_VPT] = kNaN;
      mn = fminf(mn, __uint_as_float(v[4 * NPAIR_LSB_VPT])); mx = fmaxf(mx, __uint_as_float(v[4 * NPAIR_LSB_VPT]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    if (lane == 0) { B.red_min[w] = mn; B.red_max[w] = mx; }
    __syncthreads();
    const unsigned int ns = B.n_same;                              // == cs
    float lo = B.red_min[0], hi = B.red_max[0];
#pragma unroll
    for (int k = 1; k < NPAIR_LSB_THREADS / 32; ++k) { lo = fminf(lo, B.red_min[k]); hi = fmaxf(hi, B.red_max[k]); }
    bool slow_ap = false;
    unsigned long long pos_ap = 0, pos_an = 0;
    // ---------------- AP side: the same-label list is short; warp 0 ranks it by counting ----------------
    if (want_same) {
      int err = 0;
      if (!side_position(static_cast<unsigned long long>(cs), sn_ap, pos_ap, err)) { if (tid == 0) { atomicOr(&bs->err, err); ra.posi_thr[i] = 0.f; } }
      else if (ns > NPAIR_LSEL_SCAP) slow_ap = true;
      else if (w == 0)
        store_key_of_rank([&](unsigned int t) { return f2ord(__uint_as_float(B.same[t])); }, ns, static_cast<unsigned int>(pos_ap), lane, 32,
                          &ra.posi_thr[i]);                                                                // .cu:288
    }
    // ---------------- AN side (every condition below is block-uniform) ----------------
    bool have_an = false, refine = false, by_bin = false;
    float s4 = 0.f, c0 = 0.f;
    unsigned int rank = 0;
    uint32_t boff = 0;
    if (want_diff) {
      int err = 0;
      if (!side_position(static_cast<unsigned long long>(N - 1 - cs), sn_an, pos_an, err)) { if (tid == 0) { atomicOr(&bs->err, err); ra.nega_thr[i] = 0.f; } }
      else have_an = true;
    }
    if (have_an) {
      rank = static_cast<unsigned int>(pos_an);
      // the value map: usable when it sends lo to bin >= 1 and hi to a bin the find walks (always, unless the range is empty or outside
      // what fp32 can scale -- then the key digits do the whole job)
      s4 = __fdiv_rn(4.f * NPAIR_LSB_BINS, hi - lo);
      c0 = __fmaf_rn(-lo, s4, 8388612.f);                           // 2^23 + 4: one bin of head room below lo
      const uint32_t o_lo = __float_as_uint(__fmaf_rn(lo, s4, c0)), o_hi = __float_as_uint(__fmaf_rn(hi, s4, c0));
      const bool map_ok = hi > lo && o_lo >= 0x4B000000u && o_hi >= o_lo && o_hi < 0x4B000000u + 4u * (NPAIR_LSB_HIST - 1);
      if (!map_ok) refine = true;
      else {
#pragma unroll
        for (int e = 0; e < 4 * NPAIR_LSB_VPT + 1; ++e) smem_inc_off(B.hist, lsb_off(v[e], s4, c0));
        __syncthreads();
        block_find_bin_u32<NPAIR_LSB_HIST / NPAIR_LSB_THREADS>(B, rank);
        boff = B.out[0] << 2; rank = B.out[1];
        if (B.out[2] > NPAIR_LSB_CCAP) { refine = true; by_bin = true; }
        else {
#pragma unroll
          for (int e = 0; e < 4 * NPAIR_LSB_VPT + 1; ++e)
            if (lsb_off(v[e], s4, c0) == boff) B.cand[atomicAdd(&B.n_cand, 1u)] = f2ord(__uint_as_float(v[e]));
        }
      }
      if (refine) {
        // Rare: the entries still in play (all of them, or one crowded bin) are narrowed by 11 bits of their ORDERED KEY per round, from
        // the registers: [klo, khi] always contains the wanted entry and `rank` counts inside it.
        uint32_t klo = 0xFFFFFFFFu, khi = 0u;
        auto in_play = [&](uint32_t bits) { return bits != kNaN && (!by_bin || lsb_off(bits, s4, c0) == boff); };
#pragma unroll
        for (int e = 0; e < 4 * NPAIR_LSB_VPT + 1; ++e)
          if (in_play(v[e])) { const uint32_t k = f2ord(__uint_as_float(v[e])); klo = min(klo, k); khi = max(khi, k); }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { klo = min(klo, __shfl_xor_sync(0xffffffffu, klo, o)); khi = max(khi, __shfl_xor_sync(0xffffffffu, khi, o)); }
        __syncthreads();                                            // readers of red_* / out of the steps above are done
        if (lane == 0) { B.red_klo[w] = klo; B.red_khi[w] = khi; }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < NPAIR_LSB_THREADS / 32; ++k) { klo = min(klo, B.red_klo[k]); khi = max(khi, B.red_khi[k]); }
        for (int round = 0; round < 4 && khi != klo; ++round) {
          const uint32_t range = khi - klo;
          const int shift = max(0, 32 - __clz(range) - 11);       // (range >> shift) < 2048
          for (int b = tid * 4; b < NPAIR_LSB_HIST; b += NPAIR_LSB_THREADS * 4) *reinterpret_cast<uint4*>(&B.hist[b]) = make_uint4(0u, 0u, 0u, 0u);
          __syncthreads();
#pragma unroll
          for (int e = 0; e < 4 * NPAIR_LSB_VPT + 1; ++e)
            if (in_play(v[e])) { const uint32_t k = f2ord(__uint_as_float(v[e])); if (k >= klo && k <= khi) smem_inc(&B.hist[(k - klo) >> shift]); }
          __syncthreads();
          block_find_bin_u32<NPAIR_LSB_HIST / NPAIR_LSB_THREADS>(B, rank);
          rank = B.out[1];
          klo += B.out[0] << shift;
          khi = min(khi, klo + ((shift ? (1u << shift) : 1u) - 1u));
        }
        if (tid == 0) ra.nega_thr[i] = clamp_thr(ord2f(klo));                                               // .cu:319
      }
    }
    // ---------------- the registers are free: the next row streams in while this row's pick runs ----------------
    const float* row = sim.row(i);
    if (i + static_cast<int>(gridDim.x) < row_end) load_row(i + static_cast<int>(gridDim.x));
    if (have_an && !refine) {
      __syncthreads();
      store_key_of_rank([&](unsigned int t) { return B.cand[t]; }, B.n_cand, rank, tid, NPAIR_LSB_THREADS, &ra.nega_thr[i]);   // .cu:319
    }
    if (slow_ap) {                                                 // more than 128 same-label entries: warp 0 redoes the side with plain sweeps
      __syncthreads();
      if (w == 0) { const float t = clamp_thr(ord2f(slow_select_row(row, N, lab_cols, li, self_col, 0, static_cast<unsigned int>(pos_ap), B.hist, lane))); if (lane == 0) ra.posi_thr[i] = t; }
    }
    __syncthreads();
  }
}
static constexpr int LSEL_SMEM = static_cast<int>(sizeof(LselWarp)) * NPAIR_LSEL_WARPS;
cudaError_t allow_local_select_smem() {
  return cudaFuncSetAttribute(local_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, LSEL_SMEM);
}
void launch_local_select(SimRows sim, int side_mask, float sn_ap, float sn_an, RowArrays ra, BlockScalars* bs, int sms, bool force_warp_kernel, cudaStream_t st) {
  if (!force_warp_kernel && sim.N <= NPAIR_LSB_THREADS * NPAIR_LSB_VPT * 4 && (reinterpret_cast<uintptr_t>(sim.lab_cols) & 15) == 0 && (sim.ldS & 3) == 0) {
    int grid = sms * NPAIR_LSB_MINB; if (grid > sim.rows) grid = sim.rows;
    local_select_block_kernel<<<grid, NPAIR_LSB_THREADS, 0, st>>>(sim, side_mask, sn_ap, sn_an, ra, bs);
    count_launch();
    return;
  }
  const int per_sm = (227 * 1024) / (LSEL_SMEM + 1024);
  int grid = sms * (per_sm < 1 ? 1 : per_sm);
  const int need = (sim.rows + NPAIR_LSEL_WARPS - 1) / NPAIR_LSEL_WARPS;
  if (grid > need) grid = need;
  local_select_kernel<<<grid, 32 * NPAIR_LSEL_WARPS, LSEL_SMEM, st>>>(sim, side_mask, sn_ap, sn_an, ra, bs);
  count_launch();
}

// ---- GLOBAL: the rank's whole Q x N block.  Three kernels, each finished by its last block (ticket):
//   A  digit 1 (top 11 bits of the RAW float bits; three instructions per element on the all-different-label fast path) histogram
//      over S, 64-bit global counts; the last block walks the bins in value order -> bin, rank inside, population
//   B  second sweep of S: elements of that bin only (a shift and a compare per element): digit 2 histogram of their 21-bit
//      remainders, and -- when the bin fits the candidate buffer -- the remainders are compacted (per-block staging, one global
//      atomic per flush)
//   C  digit 3 over the candidates (or, oversized bin, over S once more) -> threshold, written to all rows
// Remainders of negative floats sort descending, so they are stored complemented ("flipped"): ascending everywhere.
struct GlobalSelectBufs {
  unsigned long long* hist;   // [2][2048]
  uint32_t* cand;             // [2][cap]
  unsigned int cap;
  int world_scope;            // 1: the digit counts are exchanged between the ranks before the decision
};
#define NPAIR_GSEL_STAGE 2048

// Bin of 0-based rank r among bins 0 .. nb-1 taken in index order, bin b holding cnt(b) entries, by the block (any size that is a
// multiple of 32): every thread sums a run of bins and the one whose run holds r walks it.  Three barriers; afterwards
// s_out = {bin, rank inside it, its population} (bin == nb: r is out of range).  s_scan: 32 counts of shared memory.
// Not merged with block_find_bin_u32: holding 64-bit counts in registers the way that finder does raises global_select_kernel, which
// inlines this decision into its last block, from 55 to 58-60 registers (CUDA 12.9) in every form tried.
template <class C>
__device__ __forceinline__ void find_bin(C cnt, int nb, unsigned long long r, unsigned long long* s_scan, unsigned long long* s_out) {
  const int per = (nb + blockDim.x - 1) / blockDim.x;
  const int b0 = threadIdx.x * per, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long mine = 0;
  for (int b = b0; b < b0 + per && b < nb; ++b) mine += cnt(b);
  const unsigned long long incl = warp_incl_sum(mine, lane);
  if (lane == 31) s_scan[w] = incl;
  if (threadIdx.x == 0) s_out[0] = static_cast<unsigned long long>(nb);
  __syncthreads();
  if (w == 0) s_scan[lane] = warp_incl_sum((lane < static_cast<int>(blockDim.x >> 5)) ? s_scan[lane] : 0ull, lane);   // inclusive warp totals
  __syncthreads();
  const unsigned long long before = (w ? s_scan[w - 1] : 0ull) + incl - mine;
  if (mine && r >= before && r < before + mine) {                 // exactly one thread
    unsigned long long cum = before;
    int b = b0;
    for (; b < b0 + per && b < nb; ++b) { const unsigned long long h = cnt(b); if (cum + h > r) break; cum += h; }
    s_out[0] = static_cast<unsigned long long>(b); s_out[1] = r - cum; s_out[2] = cnt(b);
  }
  __syncthreads();
}

// Decides one digit of the GLOBAL select from the 64-bit counts in gb.hist (one block; s_scan, s_out: find_bin's shared memory)
__device__ void global_decide(int pass, bool act0, bool act1, GlobalSelectBufs gb, RowArrays ra, int Q, BlockScalars* bs,
                              unsigned long long* s_scan, unsigned long long* s_out) {
  const int shift = pass == 1 ? 10 : 0;
  const int nbits = pass == 2 ? 10 : 11;
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    if (!(side == 0 ? act0 : act1)) continue;
    const unsigned long long* gh = gb.hist + side * NPAIR_SEL_BINS;
    const int nb = 1 << nbits;
    // pass 0 counted RAW digits: they are read in value order
    find_bin([&](int o) { return __ldcg(&gh[pass == 0 ? raw_digit_of_order(o, 11) : static_cast<uint32_t>(o)]); }, nb, bs->sel_rank[side],
             s_scan, s_out);
    if (threadIdx.x == 0) {
      const int d = static_cast<int>(s_out[0]);
      if (d >= nb) { bs->err |= DERR_POS_RANGE; bs->sel_active[side] = 0; }
      else {
        bs->sel_rank[side] = s_out[1];
        if (pass == 0) { bs->sel_prefix[side] = raw_digit_of_order(static_cast<uint32_t>(d), 11) << 21; bs->sel_cnt[side] = s_out[2]; bs->cand_n[side] = 0; }
        else bs->sel_prefix[side] |= static_cast<uint32_t>(d) << shift;
        if (pass == 2) {
          const uint32_t p = bs->sel_prefix[side];
          const float thr = clamp_thr(__uint_as_float(p ^ rem_flip(p, 21)));   // .cu:303 / :334
          if (side == 0) bs->posi_global = thr; else bs->nega_global = thr;
        }
      }
    }
    __syncthreads();
  }
  for (int b = threadIdx.x; b < 2 * NPAIR_SEL_BINS; b += blockDim.x) gb.hist[b] = 0ull;
  if (pass == 2) {
    __syncthreads();
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      if (!(side == 0 ? act0 : act1) || !bs->sel_active[side]) continue;
      const float thr = side == 0 ? bs->posi_global : bs->nega_global;
      float* out = side == 0 ? ra.posi_thr : ra.nega_thr;
      for (int i = threadIdx.x; i < Q; i += blockDim.x) out[i] = thr;
    }
  }
}

__global__ void __launch_bounds__(512) global_select_kernel(const float* __restrict__ S, long long ldS, int Q, int N, const float* __restrict__ lab_rows,
                                                            const float* __restrict__ lab_cols, int self_offset, int side_mask, int pass /*0,1,2*/,
                                                            GlobalSelectBufs gb, RowArrays ra, BlockScalars* bs) {
  __shared__ unsigned int hist[2][NPAIR_SEL_BINS];
  __shared__ uint32_t stage[2][NPAIR_GSEL_STAGE];
  __shared__ unsigned int s_nst[2], s_base[2];
  __shared__ unsigned long long s_scan[32], s_out[3];
  __shared__ int s_last;
  const bool act0 = (side_mask & 1) && bs->sel_active[0], act1 = (side_mask & 2) && bs->sel_active[1];
  if (!act0 && !act1) return;
  const bool lab_aligned = (reinterpret_cast<uintptr_t>(lab_cols) & 15) == 0;
  const int shift = pass == 1 ? 10 : 0;
  const int nbits = pass == 2 ? 10 : 11;
  const uint32_t dm = (1u << nbits) - 1u;
  // sel_prefix after pass 0: raw digit << 21; after pass 1: | flipped-remainder digit << 10
  const uint32_t raw0 = bs->sel_prefix[0] >> 21, raw1 = bs->sel_prefix[1] >> 21;
  const uint32_t flip0 = rem_flip(bs->sel_prefix[0], 21), flip1 = rem_flip(bs->sel_prefix[1], 21);
  const uint32_t mid0 = (bs->sel_prefix[0] >> 10) & 0x7FFu, mid1 = (bs->sel_prefix[1] >> 10) & 0x7FFu;   // pass 2: decided second digit
  const bool comp0 = act0 && pass == 1 && bs->sel_cnt[0] <= gb.cap, comp1 = act1 && pass == 1 && bs->sel_cnt[1] <= gb.cap;   // compaction this pass
  const bool list0 = act0 && pass == 2 && bs->sel_cnt[0] <= gb.cap, list1 = act1 && pass == 2 && bs->sel_cnt[1] <= gb.cap;   // read the list this pass
  for (int b = threadIdx.x; b < 2 * NPAIR_SEL_BINS; b += blockDim.x) (&hist[0][0])[b] = 0;
  if (threadIdx.x < 2) s_nst[threadIdx.x] = 0;
  __syncthreads();
  const bool sweep0 = act0 && !list0, sweep1 = act1 && !list1;

  // one element of the bin of `side` (passes 1 and 2): its flipped remainder goes to the digit histogram / the staging list
  auto take = [&](uint32_t bits, int side) {
    const uint32_t k = (bits & 0x1FFFFFu) ^ (side == 0 ? flip0 : flip1);
    if (pass == 2 && ((k >> 10) != (side == 0 ? mid0 : mid1))) return;
    smem_inc(&hist[side][(k >> shift) & dm]);
    if (side == 0 ? comp0 : comp1) {
      const unsigned int slot = atomicAdd(&s_nst[side], 1u);
      if (slot < NPAIR_GSEL_STAGE) stage[side][slot] = k;
      else {                                                     // staging full (rare): straight to the global list
        const unsigned int g = atomicAdd(&bs->cand_n[side], 1u);
        if (g < gb.cap) gb.cand[static_cast<size_t>(side) * gb.cap + g] = k;
      }
    }
  };

  if (sweep0 || sweep1) {
    for (int i = blockIdx.x; i < Q; i += gridDim.x) {
      const SimRows sim{S, ldS, Q, N, 0, Q, lab_rows, lab_cols, self_offset};    // the rank's whole S
      const float li = lab_rows[i];
      const float* row = sim.row(i);
      // two 16-byte groups per thread in flight (S and labels): the sweeps are latency-bound otherwise
      for (int j0 = threadIdx.x * 4; j0 < N; j0 += blockDim.x * 8) {
        uint4 vq[2]; float lq[2][4];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j4 = j0 + u * blockDim.x * 4;
          if (j4 >= N) continue;
          vq[u] = __ldg(reinterpret_cast<const uint4*>(row + j4));              // row stride is a multiple of 32 floats: in bounds
          if (lab_aligned && j4 + 3 < N) { const float4 l = __ldg(reinterpret_cast<const float4*>(lab_cols + j4)); lq[u][0] = l.x; lq[u][1] = l.y; lq[u][2] = l.z; lq[u][3] = l.w; }
          else {
#pragma unroll
            for (int c = 0; c < 4; ++c) lq[u][c] = (j4 + c < N) ? __ldg(lab_cols + j4 + c) : li;
          }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
        const int j4 = j0 + u * blockDim.x * 4;
        if (j4 >= N) continue;
        const uint32_t vv[4] = {vq[u].x, vq[u].y, vq[u].z, vq[u].w};
        const float* ll = lq[u];
        const bool no_self = !sim.self_in4(i, j4);
        if (j4 + 3 < N && no_self && ll[0] != li && ll[1] != li && ll[2] != li && ll[3] != li) {     // four diff-label pairs: the common case
          if (sweep1) {
            if (pass == 0) {
#pragma unroll
              for (int c = 0; c < 4; ++c) smem_inc_off(hist[1], (vv[c] >> 19) & 0x1FFCu);
            } else if ((vv[0] >> 21) == raw1 || (vv[1] >> 21) == raw1 || (vv[2] >> 21) == raw1 || (vv[3] >> 21) == raw1) {
#pragma unroll
              for (int c = 0; c < 4; ++c) if ((vv[c] >> 21) == raw1) take(vv[c], 1);
            }
          }
        } else {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (j4 + c >= N || j4 + c == sim.self_col(i)) continue;             // the self pair is in neither list (.cu:54)
            const int side = (ll[c] == li) ? 0 : 1;
            if (!(side == 0 ? sweep0 : sweep1)) continue;
            if (pass == 0) smem_inc(&hist[side][vv[c] >> 21]);
            else if ((vv[c] >> 21) == (side == 0 ? raw0 : raw1)) take(vv[c], side);
          }
        }
        }
      }
      if (pass == 1 && (comp0 || comp1)) {                         // flush a staging area that is at least half full
        __syncthreads();
#pragma unroll
        for (int side = 0; side < 2; ++side) {
          const unsigned int n = min(s_nst[side], static_cast<unsigned int>(NPAIR_GSEL_STAGE));
          if (n >= NPAIR_GSEL_STAGE / 2) {
            if (threadIdx.x == 0) s_base[side] = atomicAdd(&bs->cand_n[side], n);
            __syncthreads();
            for (unsigned int e = threadIdx.x; e < n; e += blockDim.x)
              if (s_base[side] + e < gb.cap) gb.cand[static_cast<size_t>(side) * gb.cap + s_base[side] + e] = stage[side][e];
            __syncthreads();
            if (threadIdx.x == 0) s_nst[side] = 0;
          }
        }
        __syncthreads();
      }
    }
  }
  if (list0 || list1) {                                            // pass 2 over the compact candidate lists (flipped remainders)
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      if (!(side == 0 ? list0 : list1)) continue;
      const unsigned int n = bs->cand_n[side];
      const uint32_t mid = side == 0 ? mid0 : mid1;
      const uint32_t* cl = gb.cand + static_cast<size_t>(side) * gb.cap;
      for (unsigned int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const uint32_t k = cl[e];
        if ((k >> 10) == mid) smem_inc(&hist[side][k & dm]);
      }
    }
  }
  __syncthreads();
  if (pass == 1) {                                                 // remaining staged candidates
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      const unsigned int n = min(s_nst[side], static_cast<unsigned int>(NPAIR_GSEL_STAGE));
      if (n) {
        if (threadIdx.x == 0) s_base[side] = atomicAdd(&bs->cand_n[side], n);
        __syncthreads();
        for (unsigned int e = threadIdx.x; e < n; e += blockDim.x)
          if (s_base[side] + e < gb.cap) gb.cand[static_cast<size_t>(side) * gb.cap + s_base[side] + e] = stage[side][e];
        __syncthreads();
      }
    }
  }
  for (int b = threadIdx.x; b < 2 * NPAIR_SEL_BINS; b += blockDim.x) {
    const unsigned int h = (&hist[0][0])[b];
    if (h) atomicAdd(&gb.hist[b], static_cast<unsigned long long>(h));
  }
  // ---- last block: decide this digit (world scope: the counts are exchanged first, global_decide_kernel decides) ----
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&bs->ticket3, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x == 0) bs->ticket3 = 0;
  if (gb.world_scope) return;
  global_decide(pass, act0, act1, gb, ra, Q, bs, s_scan, s_out);
}
// world scope: sum the ranks' digit counts (same order on every rank -> identical decisions), then decide like the last block does
__global__ void __launch_bounds__(512) global_decide_kernel(const float* __restrict__ xall, int xstride, int world, int side_mask, int pass,
                                                            GlobalSelectBufs gb, RowArrays ra, int Q, BlockScalars* bs) {
  __shared__ unsigned long long s_scan[32], s_out[3];
  const bool act0 = (side_mask & 1) && bs->sel_active[0], act1 = (side_mask & 2) && bs->sel_active[1];
  if (!act0 && !act1) return;
  for (int b = threadIdx.x; b < 2 * NPAIR_SEL_BINS; b += blockDim.x) {
    unsigned long long sum = 0;
    for (int r = 0; r < world; ++r) sum += reinterpret_cast<const unsigned long long*>(xall + static_cast<long long>(r) * xstride)[b];
    gb.hist[b] = sum;
  }
  __syncthreads();
  global_decide(pass, act0, act1, gb, ra, Q, bs, s_scan, s_out);
}
void launch_global_select_pass(SimRows sim, int side_mask, int pass, RowArrays ra, unsigned long long* hist, uint32_t* cand, unsigned int cand_cap,
                               int world_scope, BlockScalars* bs, int sms, cudaStream_t st) {
  assert(sim.row0 == 0 && sim.rows == sim.Q && "the GLOBAL select sweeps the rank's whole S");
  int grid = sms * 4; if (grid > sim.rows) grid = sim.rows;
  GlobalSelectBufs gb; gb.hist = hist; gb.cand = cand; gb.cap = cand_cap; gb.world_scope = world_scope;
  // positional arguments, from which the kernel builds its view of the whole S: as a view parameter it compiles to other, slower code
  global_select_kernel<<<grid, 512, 0, st>>>(sim.S, sim.ldS, sim.Q, sim.N, sim.lab_rows, sim.lab_cols, sim.col0, side_mask, pass, gb, ra, bs);
  count_launch();
}
void launch_global_decide(const float* xall, int xstride, int world, int side_mask, int pass, RowArrays ra, int Q, unsigned long long* hist,
                          uint32_t* cand, unsigned int cand_cap, BlockScalars* bs, cudaStream_t st) {
  GlobalSelectBufs gb; gb.hist = hist; gb.cand = cand; gb.cap = cand_cap; gb.world_scope = 1;
  global_decide_kernel<<<1, 512, 0, st>>>(xall, xstride, world, side_mask, pass, gb, ra, Q, bs);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// The forward row pass: one streaming read of S per row computes everything the reference spreads over
// GetSampledPairMtx (.cu:69-122), the count gemvs (.cu:355-360), Minus_Querywise_Maxval (.cu:124-156), the
// masked sums (.cu:373-380), ManipulateDIVandLOG (.cu:158-171) and GetRetrivePerformance (.cu:173-206).
// Retrieval uses the sort-free equivalence of SURVEY.md 9.4 Q11: with p* = max E over same-label non-self
// columns and c = #{non-self j : E_j >= p*},  hit_k  <=>  c <= min(k, N-2).
// --------------------------------------------------------------------------------------------
// Smallest float s (as an ordered key) with expf(s - max_all) >= pstar, searched downward from the best positive.
// Lets the retrieval count compare similarities instead of exponentials, so expf is only evaluated for SELECTED pairs.
__device__ __forceinline__ float retrieval_cut(float maxw, float max_all, int lane) {
  const float pstar = expf(maxw - max_all);
  if (!(pstar > 0.f)) return -INFINITY;                         // underflow: every entry ties with the best positive
  uint32_t base = f2ord(maxw), last_ok = base;
  for (int it = 0; it < 8; ++it) {                             // 256 ulps cover the flat steps of expf for |s-max| < ~80
    const uint32_t kc = base - static_cast<uint32_t>(lane);
    const bool ok = (kc <= base) && (expf(ord2f(kc) - max_all) >= pstar);
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    const int T = (bal == 0xffffffffu) ? 32 : (__ffs(~bal) - 1);
    if (T > 0) last_ok = base - static_cast<uint32_t>(T - 1);
    if (T < 32) return ord2f(last_ok);
    if (base < 64u) return ord2f(last_ok);
    base -= 32u;
  }
  // long flat step (denormal exponentials): bisection on the ordered keys, monotone expf assumed
  uint32_t lo = f2ord(-FLT_MAX), hi = last_ok;                 // invariant: hi satisfies
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (expf(ord2f(mid) - max_all) >= pstar) hi = mid; else lo = mid + 1u;
  }
  return ord2f(hi);
}

// 16-byte streaming load: read-only path, no L1 allocation (S is read exactly once by this kernel)
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

// One warp per anchor row, branch-free hot loop (12 instructions per element): one retrieval-count compare, one label
// compare, ONE selection compare with sign/threshold picked by the label predicate, a 2-instruction exponential, and two
// accumulations (T = A + B for every selected pair, A under the same-label predicate).
__device__ __forceinline__ void lse_elem(float sv, float lab, float li, float scut, float m2, float sgn_p, float thr_p,
                                         float sgn_n, float thr_n, float& A, float& T, int& c) {
  c += (sv >= scut) ? 1 : 0;                                  // == (exp(sv-max_all) >= exp(maxw-max_all)), SURVEY Q11
  const float e = fast_exp_m2(sv, m2);                        // .cu:130-131
  const bool same = (lab == li);
  const float key = sv * (same ? sgn_p : sgn_n);              // .cu:79-120 as one compare  +-s <= thr'
  const float es = (key <= (same ? thr_p : thr_n)) ? e : 0.f;
  T += es;
  if (same) A += es;
}

// The tops of `rows` rows (loss, retrieval ratios, asum) and the error word from the reduction, in order from record 0, of n records
// `stride` floats apart (world scope: one per rank, rows = N; per rank: n = 1, rows = Q), published to the host with the sequence number
__device__ __forceinline__ void publish_tops(const TopSums* recs, int n, long long stride, long long rows, int num_tops, TopsBlock* out,
                                             unsigned int seq) {
  double ls = recs[0].loss_sum, asum = recs[0].asum;
  long long h[3] = {recs[0].hits[0], recs[0].hits[1], recs[0].hits[2]};
  int err = recs[0].err;
  for (int r = 1; r < n; ++r) {
    const TopSums& t = rank_record(recs, stride, r);
    ls += t.loss_sum; h[0] += t.hits[0]; h[1] += t.hits[1]; h[2] += t.hits[2]; asum += t.asum; err |= t.err;
  }
  float tops[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  tops[0] = static_cast<float>(ls) / static_cast<float>(-rows);                               // .cu:384-385
  for (int t = 1; t <= num_tops - 2 && t <= 3; ++t) tops[t] = static_cast<float>(h[t - 1]) / static_cast<float>(rows);   // .cu:205
  tops[num_tops - 1] = static_cast<float>(asum) / static_cast<float>(rows);                   // .cu:400-401 (always the LAST top)
  for (int t = 0; t < 5; ++t) out->tops[t] = tops[t];
  out->err = err;
  __threadfence_system();
  *reinterpret_cast<volatile unsigned int*>(&out->seq) = seq;     // the tops are visible on the host before the sequence number
}

// The Q rows' TopSums by one block, published (xout == NULL) or written to *xout (world scope: the rank's record for the exchange).
// The summation order depends on the block size only (threads stride the rows, then warps in order), so a separate launch with the
// same size gives the same bits.
__device__ __forceinline__ void lse_finalize_block(int Q, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* __restrict__ tops,
                                                   TopSums* __restrict__ xout, unsigned int seq) {
  const int lane = threadIdx.x & 31;
  __shared__ double s_l[8];
  __shared__ int s_h[3][8];
  double ls = 0.0; int h[3] = {0, 0, 0};
  // FU rows per thread and trip, all 4*FU loads issued before the first use: with one row per trip this tail was a chain of 32 L2
  // latencies at Q = 8192 (~20 us of the row pass).  The per-thread summation order (r ascending) is unchanged.
  constexpr int FU = 8;
  for (int r0 = threadIdx.x; r0 < Q; r0 += FU * blockDim.x) {
    float lv[FU]; int h0[FU], h1[FU], h2[FU];
#pragma unroll
    for (int u = 0; u < FU; ++u) {
      const int r = r0 + u * blockDim.x;
      const bool ok = r < Q;
      lv[u] = ok ? __ldcg(&ra.logv[r]) : 0.f;
      h0[u] = ok ? __ldcg(&ra.hits[r]) : 0; h1[u] = ok ? __ldcg(&ra.hits[Q + r]) : 0; h2[u] = ok ? __ldcg(&ra.hits[2 * Q + r]) : 0;
    }
#pragma unroll
    for (int u = 0; u < FU; ++u) { ls += lv[u]; h[0] += h0[u]; h[1] += h1[u]; h[2] += h2[u]; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ls += __shfl_xor_sync(0xffffffffu, ls, o);
    h[0] += __shfl_xor_sync(0xffffffffu, h[0], o); h[1] += __shfl_xor_sync(0xffffffffu, h[1], o); h[2] += __shfl_xor_sync(0xffffffffu, h[2], o);
  }
  const int w = threadIdx.x >> 5;
  if (lane == 0) { s_l[w] = ls; s_h[0][w] = h[0]; s_h[1][w] = h[1]; s_h[2][w] = h[2]; }
  __syncthreads();
  if (threadIdx.x == 0) {
    TopSums s{0.0, {0, 0, 0}, bs->asum, bs->err};
    for (int k = 0; k < (blockDim.x >> 5); ++k) { s.loss_sum += s_l[k]; s.hits[0] += s_h[0][k]; s.hits[1] += s_h[1][k]; s.hits[2] += s_h[2][k]; }
    bs->ticket = 0;
    if (xout) *xout = s;
    else publish_tops(&s, 1, 0, Q, num_tops, tops, seq);
  }
}

// The last block to finish also performs the job of the old finalize kernel (loss, retrieval ratios, asum, error word), unless
// `finalize` is 0 (row-block mode: lse_finalize_kernel runs once after the last block of rows).
#ifndef NPAIR_LSE_U
#define NPAIR_LSE_U 4            // 16-byte loads in flight per lane and array (S, labels)
#endif
#ifndef NPAIR_LSE_MINB
#define NPAIR_LSE_MINB 3
#endif
__global__ void __launch_bounds__(256, NPAIR_LSE_MINB) lse_rows_kernel(const __grid_constant__ SimRows sim, MiningParams mp, RowArrays ra, BlockScalars* bs,
                                                       int num_tops, TopsBlock* __restrict__ tops, float log2_world,
                                                       TopSums* __restrict__ xout /*world scope: this rank's tops sums, else NULL*/,
                                                       int wpr /*warps per row: 1, 2, 4 or 8 (few rows per rank: keep the SMs full)*/,
                                                       unsigned int seq /*written behind the tops: the host polls it*/, int finalize) {
  const int lane = threadIdx.x & 31;
  __shared__ float s_pA[8], s_pT[8];
  __shared__ int s_pc[8];
  // NPAIR_LSE_REV: walk the rows from the last to the first.  The similarity GEMM produced the high row blocks last, so
  // their tiles are the ones still resident in the 126 MB L2 when this kernel starts.
#ifndef NPAIR_LSE_REV
#define NPAIR_LSE_REV 1
#endif
  const int blk = NPAIR_LSE_REV ? static_cast<int>(gridDim.x - 1 - blockIdx.x) : static_cast<int>(blockIdx.x);
  const int wib = threadIdx.x >> 5;
  const int il = blk * ((blockDim.x >> 5) / wpr) + wib / wpr;  // row of the launch
  const int i = sim.row0 + il;                                  // row of the rank
  const int Q = sim.Q, N = sim.N;
  const float* lab_cols = sim.lab_cols;
  const int part = wib % wpr;                                   // this warp's column segment of the row
  float A = 0.f, T = 0.f; int c = 0;
  float m2 = 0.f, thr_p = 0.f, thr_n = 0.f, li = 0.f; int cs = 0;
  if (il < sim.rows) {
    // the first block of this warp's segment is requested before anything else: the per-row set-up below (dependent loads of the row
    // statistics, the retrieval cut's expf search) then runs under the DRAM latency instead of in front of it
    constexpr int U = NPAIR_LSE_U;
    const float* row = sim.row(i);
    // this warp's segment [c_lo, c_hi) of the row: multiples of 512 columns
    const int seg = ((N + wpr - 1) / wpr + 128 * U - 1) / (128 * U) * (128 * U);
    const int c_lo = min(N, part * seg), c_hi = min(N, c_lo + seg);
    const int n_full = c_lo + (c_hi - c_lo) / (128 * U) * (128 * U);
    const float4* srow4 = reinterpret_cast<const float4*>(row + c_lo) + lane;
    const float4* lab4 = reinterpret_cast<const float4*>(lab_cols + c_lo) + lane;
    const bool lab_aligned = (reinterpret_cast<uintptr_t>(lab_cols) & 15) == 0;
    const bool fast = lab_aligned && c_lo < n_full;
    float4 v[U], vn[U];
    if (fast) {
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = ldg_stream(srow4 + 32 * u);
    }
    li = __ldg(sim.lab_rows + i);
    const int self_col = sim.self_col(i);
    const float max_all = ord2f(ra.st_maxall[i]);
    m2 = max_all * LOG2E;
    // GLOBAL-region thresholds are block-wide scalars (finish_thresholds / global_decide); LOCAL ones are per row
    const float posi = mp.ap_region == REGION_GLOBAL ? bs->posi_global : ra.posi_thr[i];
    const float nega = mp.an_region == REGION_GLOBAL ? bs->nega_global : ra.nega_thr[i];
    if (lane == 0 && part == 0) { ra.posi_thr[i] = posi; ra.nega_thr[i] = nega; }   // kept per row for inspection (npair_debug_read)
    const float tp = posi + mp.margin_ident;                    // fp32 add as in .cu:81
    const float tn = nega + mp.margin_diff;                     // .cu:102
    const float sgn_p = ap_sign(mp.ap_method), sgn_n = an_sign(mp.an_method);
    thr_p = ap_thr(tp, mp.ap_method); thr_n = an_thr(tn, mp.an_method);
    cs = ra.cnt_same[i];
    const float scut = cs > 0 ? retrieval_cut(ord2f(ra.st_maxw[i]), max_all, lane) : INFINITY;
    // ---- full 512-column blocks: unguarded 128-bit loads (4 in flight per lane for S, 4 for the labels) ----
    int base = c_lo;
    if (fast) {
      // software pipeline: the 16-byte loads of block k+1 (streamed past the L1: every byte of S is used once) are in flight while
      // block k is evaluated; the labels (32 KB shared by every row) come from the L1 when they are needed
      for (; base < n_full; base += 128 * U, srow4 += 32 * U, lab4 += 32 * U) {
        const bool more = base + 128 * U < n_full;
        if (more) {
#pragma unroll
          for (int u = 0; u < U; ++u) vn[u] = ldg_stream(srow4 + 32 * U + 32 * u);
        }
        float4 l[U];
#pragma unroll
        for (int u = 0; u < U; ++u) l[u] = __ldg(lab4 + 32 * u);
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int j4 = base + u * 128 + lane * 4;
          const float vv[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
          const float ll[4] = {l[u].x, l[u].y, l[u].z, l[u].w};
          const bool no_self = !sim.self_in4(i, j4);
          if (no_self && ll[0] != li && ll[1] != li && ll[2] != li && ll[3] != li) {
            // four diff-label pairs (all but ~cnt_same/4 groups of a row): no label-dependent selects, 8 instructions per pair
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              c += (vv[q] >= scut) ? 1 : 0;
              const float e = fast_exp_m2(vv[q], m2);
              if (vv[q] * sgn_n <= thr_n) T += e;
            }
          } else if (no_self) {
#pragma unroll
            for (int q = 0; q < 4; ++q) lse_elem(vv[q], ll[q], li, scut, m2, sgn_p, thr_p, sgn_n, thr_n, A, T, c);
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q)
              if (j4 + q != self_col) lse_elem(vv[q], ll[q], li, scut, m2, sgn_p, thr_p, sgn_n, thr_n, A, T, c);
          }
        }
        if (more) {
#pragma unroll
          for (int u = 0; u < U; ++u) v[u] = vn[u];
        }
      }
    }
    // ---- ragged tail (and the whole row when the label pointer is not 16-byte aligned) ----
    for (; base < c_hi; base += 512) {
#pragma unroll 1
      for (int u = 0; u < 4; ++u) {
        const int j4 = base + u * 128 + lane * 4;
        if (j4 >= c_hi) continue;
        const float4 v4 = *reinterpret_cast<const float4*>(row + j4);      // row stride ldS is a multiple of 32: in bounds
        const float vv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (j4 + q < c_hi && j4 + q != self_col) lse_elem(vv[q], lab_cols[j4 + q], li, scut, m2, sgn_p, thr_p, sgn_n, thr_n, A, T, c);
      }
    }
    A = warp_sum(A); T = warp_sum(T); c = warp_sum_i(c);
  }
  if (wpr > 1) {                                                // the row's segments, added in segment order by its first warp
    if (lane == 0) { s_pA[wib] = A; s_pT[wib] = T; s_pc[wib] = c; }
    __syncthreads();
    if (part == 0) {
      A = 0.f; T = 0.f; c = 0;
      for (int q = 0; q < wpr; ++q) { A += s_pA[wib + q]; T += s_pT[wib + q]; c += s_pc[wib + q]; }
    }
  }
  if (il < sim.rows && part == 0) {
    if (lane == 0) {
      ra.A[i] = A; ra.T[i] = T;                                 // T = A + B (.cu:380)
      ra.logv[i] = (A == 0.f || T == 0.f) ? 0.f : logf(A / T);  // .cu:162-169
      const int lim = N - 2;
      ra.hits[i] = (cs > 0 && c <= min(1, lim)) ? 1 : 0;
      ra.hits[Q + i] = (cs > 0 && c <= min(5, lim)) ? 1 : 0;
      ra.hits[2 * Q + i] = (cs > 0 && c <= min(10, lim)) ? 1 : 0;
      const float invA = A == 0.f ? 0.f : 1.f / A;              // Get_Query_Diff_Part zero rules (.cu:410-415)
      const float invT = T == 0.f ? 0.f : 1.f / T;
      const float cA = invT - invA;
      ra.rowrec[i] = RowRecord::make(T == 0.f ? INFINITY : m2 + log2f(T) + log2_world, thr_n, m2, li, thr_p, cA, invT);
    }
  }
  if (!finalize) return;
  // ---- grid-level completion: the last block reduces the row results (fixed order -> deterministic) ----
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&bs->ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  lse_finalize_block(Q, ra, bs, num_tops, tops, xout, seq);
}
__global__ void lse_finalize_kernel(int Q, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* __restrict__ tops, unsigned int seq) {
  lse_finalize_block(Q, ra, bs, num_tops, tops, nullptr, seq);
}
// Launch shape of the row pass, from the rank's row count Q (never from a row block's: the warps per row set the summation order
// of A and T, the block size that of the finaliser).
static void lse_shape(int Q, int N, int* wpr_out, int* threads_out) {
  // few rows per rank (anchor sharding over many GPUs): several warps share a row so that every SM still holds ~32 warps
  int wpr = 1;
  while (wpr < 8 && static_cast<long long>(Q) * wpr < 4096 && N / (2 * wpr) >= 512) wpr *= 2;
  // measured on one rank's strip of a sharded HL job (tests/tune_rank.py, N = 8192): Q = 1024: 2 warps per row 18.6 us, 4: 22.7, 8: 25.5;
  // Q = 2048: 2: 29.8, 8: 37.1 -- beyond two warps the per-warp set-up outweighs the fuller SMs
  if (Q >= 1024 && wpr > 2) wpr = 2;
  // (measured: splitting rows over two warps at Q = 8192 to even out the 2.31 waves of one-warp-per-row blocks is slower, 80.6 vs 77 us)
#ifdef NPAIR_LSE_WPR_FORCE      // tuning builds only
  wpr = NPAIR_LSE_WPR_FORCE;
#endif
  *wpr_out = wpr;
  if (wpr > 1) { *threads_out = 256; return; }
  // 8 warps per block, 4 blocks per SM.  Measured at Q = 8192 (1.73 waves): 7 warps (1.98 waves, less idle tail) is SLOWER
  // (81.3 vs 78.7 us; 6: 83.7, 5: 87.6) -- the pass is latency-bound, more resident warps win.  NPAIR_LSE_WPB overrides.
  int wpb = 8;
  while (wpb > 1 && (Q + wpb - 1) / wpb < 296) wpb >>= 1;     // keep >= 2 blocks per SM when the rank has few rows
  *threads_out = wpb * 32;
}
void launch_lse_rows(SimRows sim, MiningParams mp, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* tops_dev, int world, TopSums* xout,
                     unsigned int seq, bool finalize, cudaStream_t st) {
  int wpr = 1, threads = 256;
  lse_shape(sim.Q, sim.N, &wpr, &threads);
  const int rows_per_blk = threads / 32 / wpr;
  const int grid = (sim.rows + rows_per_blk - 1) / rows_per_blk;
  lse_rows_kernel<<<grid, threads, 0, st>>>(sim, mp, ra, bs, num_tops, tops_dev, xout ? 0.f : log2f(static_cast<float>(world)), xout, wpr, seq,
                                            finalize ? 1 : 0);
  count_launch();
}
void launch_lse_finalize(int Q, int N, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* tops_dev, unsigned int seq, cudaStream_t st) {
  int wpr = 1, threads = 256;
  lse_shape(Q, N, &wpr, &threads);
  lse_finalize_kernel<<<1, threads, 0, st>>>(Q, ra, bs, num_tops, tops_dev, seq);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// Backward weight builder: replaces Get_Query_Diff_Part x3 (.cu:405-419, :438-446).  The reference
// materialises W1,W2,W3 in fp32 and runs six GEMMs; here one pass over S produces the unit gradient
// weight   g'(i,c) = sel(i,c) * expf(S[i,c]-max_all_i) * (same ? 1/T_i - 1/A_i : 1/T_i)     ( = -W1+W2+W3 )
// directly as split 2-byte operand tiles for the tensor-core GEMM:
//   world == 1 :  H[j][m]  = g'(j,m) + g'(m,j)            dX = (lw/Q)/2 * H . X        (.cu:448-497 folded)
//   world  > 1 :  H[j][m]  = g'(j,m)  and  HT[m][j] = g'(j,m)
//                 local = H . X_total ,  total = HT . X_local , then reduce-scatter and blend (.cu:462-497)
// --------------------------------------------------------------------------------------------
struct RowScal { float maxall, tp, tn, cA, cT, lab; };   // maxall: max_all*log2e; tp/tn: ap_thr / an_thr transformed thresholds
// A row's scalars from its record, the weight factors scaled by w.  No record (no such row): the thresholds -inf select nothing.
__device__ __forceinline__ RowScal row_scal(const RowRecord* rec, float w) {
  if (!rec) return RowScal{0.f, -INFINITY, -INFINITY, 0.f, 0.f, 0.f};
  const RowRecord r = *rec;
  return RowScal{r.m2(), r.thr_p(), r.thr_n(), r.cA() * w, r.cT() * w, r.label()};
}

// r.maxall holds max_all * log2(e) (see lse_rows_kernel)
__device__ __forceinline__ float gprime(float sv, bool same, const RowScal& r, float sgn_p, float sgn_n) {
  const float e = fast_exp_m2(sv, r.maxall);
  const float key = sv * (same ? sgn_p : sgn_n);
  return (key <= (same ? r.tp : r.tn)) ? e * (same ? r.cA : r.cT) : 0.f;
}

// four consecutive weights -> NS pieces, one 8-byte store per piece
template <int PREC>
__device__ __forceinline__ void store_quad(uint16_t* __restrict__ base, long long piece_stride, long long off, const float g[4]) {
  constexpr int NS = SPLIT_FORMATS[PREC].pieces;
  if (g[0] == 0.f && g[1] == 0.f && g[2] == 0.f && g[3] == 0.f) {          // the common case under margin mining
#pragma unroll
    for (int s = 0; s < NS; ++s) *reinterpret_cast<uint2*>(base + s * piece_stride + off) = make_uint2(0u, 0u);
    return;
  }
  uint16_t p[4][3];
#pragma unroll
  for (int e = 0; e < 4; ++e) split3<PREC>(g[e], p[e][0], p[e][1], p[e][2]);
#pragma unroll
  for (int s = 0; s < NS; ++s)
    *reinterpret_cast<uint2*>(base + s * piece_stride + off) =
        make_uint2(static_cast<uint32_t>(p[0][s]) | (static_cast<uint32_t>(p[1][s]) << 16), static_cast<uint32_t>(p[2][s]) | (static_cast<uint32_t>(p[3][s]) << 16));
}

// 64 x 64 tiles, 256 threads; thread (tr = t/16, tc = t%16) owns the 4 x 4 micro-tile rows 4tr.., columns 4tc.. :
// one 16-byte load per row of the micro-tile, one 8-byte store per row and operand piece -- every request covers whole
// sectors, nothing is transposed.
// SYM (world == 1): the similarity GEMM wrote a bitwise symmetric S (EPI_SYM), so
//     H[j][m] = g'(S[j][m]; row j) + g'(S[j][m]; row m)                       (= G + G^T, .cu:448-497 folded)
//   needs only the row scalars of BOTH indices, which are local when world == 1.
// !SYM (world > 1): H[j][m] = g'(j,m) and the transposed copy HT[m][j] (micro-tile transposed in registers).
// MODE BW_ROWSCAL (world > 1): the similarity GEMM is bitwise symmetric ACROSS ranks (K-concatenated operands), so the
//   transposed term G[m][j] of row m on another rank is evaluated here from S[j][m] and row m's all-gathered scalars:
//     H[j][m] = g'(S[j][m]; row j) + (1/world) g'(S[j][m]; row m)          -- no N x D reduce-scatter (.cu:455-497)
template <int PREC, int MODE>
__global__ void __launch_bounds__(256, 4) build_weights_kernel(const __grid_constant__ SimRows sim, float inv_world, const RowRecord* __restrict__ rs_total,
                                                            MiningParams mp, RowArrays ra,
                                                            uint16_t* __restrict__ H, long long ldH, uint16_t* __restrict__ HT, long long ldHT) {
  constexpr bool SYM = (MODE != BW_SPLIT);      // both symmetric modes add the row-m term
  constexpr int TS = 64;
  const int Q = sim.Q, N = sim.N;
  const int ta = blockIdx.y, tb = blockIdx.x;
  __shared__ RowScal sc_a[TS], sc_b[TS];
  const int a0 = ta * TS, b0 = tb * TS;
  const int t = threadIdx.x, tr = t >> 4, tc = t & 15;
  const float sgn_p = ap_sign(mp.ap_method), sgn_n = an_sign(mp.an_method);
  if (t < TS) {
    sc_a[t] = row_scal(a0 + t < Q ? ra.rowrec + a0 + t : nullptr, 1.f);
  } else if (t < 2 * TS) {
    const int mm = t - TS, m = b0 + mm;
    if (MODE == BW_SYM) {   // world == 1: column m is also a local row
      sc_b[mm] = row_scal(m < Q ? ra.rowrec + m : nullptr, 1.f);
    } else if (MODE == BW_ROWSCAL) {   // the world's records; the 1/world of .cu:474 folded into the weights
      sc_b[mm] = row_scal(m < N ? rs_total + m : nullptr, inv_world);
    } else {
      RowScal r = row_scal(nullptr, 1.f);
      if (m < N) r.lab = sim.lab_cols[m];
      sc_b[mm] = r;
    }
  }
  __syncthreads();
  const int ja0 = a0 + 4 * tr, mb0 = b0 + 4 * tc;       // my rows of block a, my columns of block b
  RowScal rb4[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) rb4[e] = sc_b[4 * tc + e];
  // block-uniform fast path: tile fully inside the matrix and not touching the self-pair diagonal
  const bool interior = (a0 + TS <= Q) && (b0 + TS <= N) && (sim.self_col(a0) + TS <= b0 || b0 + TS <= sim.self_col(a0));
  const long long psH = static_cast<long long>(Q) * ldH;
  float gT[4][4];                                        // BW_SPLIT: transposed copy for HT
  float4 v4[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {                          // all four 16-byte loads in flight before the arithmetic
    v4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ja0 + i < Q && mb0 < N) v4[i] = *reinterpret_cast<const float4*>(sim.row(ja0 + i) + mb0);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const RowScal rsa = sc_a[4 * tr + i];
    const float sv[4] = {v4[i].x, v4[i].y, v4[i].z, v4[i].w};
    float g[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = ja0 + i, m = mb0 + e;
      float x = 0.f;
      if (interior || (j < Q && m < N && m != sim.self_col(j))) {
        const bool same = rsa.lab == rb4[e].lab;
        x = gprime(sv[e], same, rsa, sgn_p, sgn_n);
        if (SYM) x += gprime(sv[e], same, rb4[e], sgn_p, sgn_n);
      }
      g[e] = x;
      if (!SYM) gT[e][i] = x;
    }
    if (ja0 + i < Q && mb0 < ldH) store_quad<PREC>(H, psH, static_cast<long long>(ja0 + i) * ldH + mb0, g);
  }
  if (!SYM) {
    const long long psT = static_cast<long long>(N) * ldHT;
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (mb0 + e < N && ja0 < ldHT) store_quad<PREC>(HT, psT, static_cast<long long>(mb0 + e) * ldHT + ja0, gT[e]);   // rows beyond Q are zero
  }
}
void launch_build_weights(SimRows sim, int world, int mode, const RowRecord* rs_total, MiningParams mp, RowArrays ra, int prec,
                          uint16_t* H, long long ldH, uint16_t* HT, long long ldHT, cudaStream_t st) {
  assert(sim.row0 == 0 && sim.rows == sim.Q && "the weight builder sweeps the rank's whole S");
  dim3 grid((sim.N + 63) / 64, (sim.Q + 63) / 64);
  const float inv_world = 1.f / static_cast<float>(world);
  with_prec(prec, [&](auto P) {
    auto kernel = mode == BW_SYM ? build_weights_kernel<P, BW_SYM> : mode == BW_ROWSCAL ? build_weights_kernel<P, BW_ROWSCAL>
                                                                                        : build_weights_kernel<P, BW_SPLIT>;
    kernel<<<grid, 256, 0, st>>>(sim, inv_world, rs_total, mp, ra, H, ldH, HT, ldHT);
  });
  count_launch();
}

// --------------------------------------------------------------------------------------------
// L2Normalize producer (usage/def.prototxt:115-120; the layer's source is not in the reference tree, so the semantics are
// stated here): y = x / ||x||_2 per sample, a zero row stays zero; backward dx = (dy - y (y . dy)) / ||x||.
// One warp per row, 16-byte loads, fixed summation order (lane-strided partial sums, then the shuffle tree).
// --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) l2norm_fwd_kernel(const float* __restrict__ x, int rows, int dim, float* __restrict__ y,
                                                         float* __restrict__ inv_norm) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* xr = x + static_cast<long long>(r) * dim;
  float* yr = y + static_cast<long long>(r) * dim;
  // dim % 4 == 0: each lane sums groups of 4 features (16-byte loads when both pointers allow, otherwise 4-byte loads in the same
  // order, so y does not depend on where x starts); else lane-strided features
  const bool quad = (dim & 3) == 0;
  const bool vec = quad && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  float ss = 0.f;
  if (vec) for (int d = lane * 4; d < dim; d += 128) { const float4 v = *reinterpret_cast<const float4*>(xr + d); ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss); }
  else if (quad) for (int d = lane * 4; d < dim; d += 128) for (int e = 0; e < 4; ++e) ss = fmaf(xr[d + e], xr[d + e], ss);
  else for (int d = lane; d < dim; d += 32) ss = fmaf(xr[d], xr[d], ss);
  ss = warp_sum(ss);
  const float nrm = sqrtf(ss);
  const float inv = nrm > 0.f ? 1.f / nrm : 0.f;
  if (lane == 0 && inv_norm) inv_norm[r] = inv;
  if (vec) for (int d = lane * 4; d < dim; d += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + d);
    *reinterpret_cast<float4*>(yr + d) = nrm > 0.f ? make_float4(v.x / nrm, v.y / nrm, v.z / nrm, v.w / nrm) : make_float4(0.f, 0.f, 0.f, 0.f);
  } else for (int d = lane; d < dim; d += 32) yr[d] = nrm > 0.f ? xr[d] / nrm : 0.f;
}
__global__ void __launch_bounds__(256) l2norm_bwd_kernel(const float* __restrict__ y, const float* __restrict__ inv_norm, const float* __restrict__ dy,
                                                         int rows, int dim, float* __restrict__ dx) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* yr = y + static_cast<long long>(r) * dim;
  const float* gr = dy + static_cast<long long>(r) * dim;
  float* dr = dx + static_cast<long long>(r) * dim;
  const bool quad = (dim & 3) == 0;            // as in l2norm_fwd_kernel: the summation order depends on dim only
  const bool vec = quad && ((reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0;
  float dot = 0.f;
  if (vec) for (int d = lane * 4; d < dim; d += 128) {
    const float4 a = *reinterpret_cast<const float4*>(yr + d), g = *reinterpret_cast<const float4*>(gr + d);
    dot = fmaf(a.x, g.x, dot); dot = fmaf(a.y, g.y, dot); dot = fmaf(a.z, g.z, dot); dot = fmaf(a.w, g.w, dot);
  } else if (quad) {
    for (int d = lane * 4; d < dim; d += 128) for (int e = 0; e < 4; ++e) dot = fmaf(yr[d + e], gr[d + e], dot);
  } else for (int d = lane; d < dim; d += 32) dot = fmaf(yr[d], gr[d], dot);
  dot = warp_sum(dot);
  const float inv = inv_norm[r];
  if (vec) for (int d = lane * 4; d < dim; d += 128) {
    const float4 a = *reinterpret_cast<const float4*>(yr + d), g = *reinterpret_cast<const float4*>(gr + d);
    *reinterpret_cast<float4*>(dr + d) = make_float4((g.x - a.x * dot) * inv, (g.y - a.y * dot) * inv, (g.z - a.z * dot) * inv, (g.w - a.w * dot) * inv);
  } else for (int d = lane; d < dim; d += 32) dr[d] = (gr[d] - yr[d] * dot) * inv;
}
// world scope: tops from the ranks' sums, normalised by the world's N (identical on every rank)
__global__ void tops_world_kernel(const TopSums* __restrict__ xall, int xstride, int world, long long N, int num_tops, TopsBlock* __restrict__ tops,
                                  unsigned int seq) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  publish_tops(xall, world, xstride, N, num_tops, tops, seq);
}
void launch_tops_world(const float* xall, int xstride, int world, long long N, int num_tops, TopsBlock* tops_dev, unsigned int seq, cudaStream_t st) {
  tops_world_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const TopSums*>(xall), xstride, world, N, num_tops, tops_dev, seq);
  count_launch();
}

void launch_l2norm_fwd(const float* x, int rows, int dim, float* y, float* inv_norm, cudaStream_t st) {
  l2norm_fwd_kernel<<<(rows + 7) / 8, 256, 0, st>>>(x, rows, dim, y, inv_norm);
  count_launch();
}
void launch_l2norm_bwd(const float* y, const float* inv_norm, const float* dy, int rows, int dim, float* dx, cudaStream_t st) {
  l2norm_bwd_kernel<<<(rows + 7) / 8, 256, 0, st>>>(y, inv_norm, dy, rows, dim, dx);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// retrieval evaluation (DESIGN 8; not part of the reference layer): operand preparation of two matrices and the best-positive cut
// --------------------------------------------------------------------------------------------
// max|x| over the queries and the gallery (g == NULL: the gallery is the query set) into *absmax_bits, which is pre-zeroed (the bits
// of non-negative floats order like the floats; NaN is skipped by fmaxf), and the reset of the per-query statistics.
__global__ void __launch_bounds__(256) eval_prep_kernel(const float* __restrict__ q, long long nq_el, const float* __restrict__ g, long long ng_el,
                                                        unsigned int* absmax_bits, RowArrays ra, int nq) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (absmax_bits) {
    float mx = 0.f;
    for (long long i = t0; i < nq_el; i += stride) mx = fmaxf(mx, fabsf(__ldg(q + i)));
    if (g) for (long long i = t0; i < ng_el; i += stride) mx = fmaxf(mx, fabsf(__ldg(g + i)));
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0 && mx > 0.f) atomicMax(absmax_bits, __float_as_uint(mx));
  }
  for (long long i = t0; i < nq; i += stride) reset_row_stats(ra, i);
}
void launch_eval_prep(const float* q, long long nq_el, const float* g, long long ng_el, unsigned int* absmax_bits, RowArrays ra, int nq,
                      int sms, cudaStream_t st) {
  const long long work = absmax_bits ? (nq_el > ng_el ? nq_el : ng_el) / 16 : nq;   // threads: ~16 elements each
  long long nb = (work + 255) / 256;
  nb = nb < 1 ? 1 : (nb > 8 * sms ? 8 * sms : nb);
  eval_prep_kernel<<<static_cast<int>(nb), 256, 0, st>>>(q, nq_el, g, ng_el, absmax_bits, ra, nq);
  count_launch();
}

// Rows of x to one side of the K-concatenated operands of the similarity GEMM (side_b = 0: the A format of the queries, 1: the B format
// of the gallery), through the layer's store_kcat_row.  Thread = 8 features of one row.  The pre-scale is the layer's rule applied to
// max|x| over both sets: `absmax` when the caller gives it (>= 0), else *absmax_bits.
template <int PREC>
__global__ void __launch_bounds__(256) eval_split_kernel(const float* __restrict__ x, int rows, int D, long long Dp, int side_b, float absmax,
                                                         const unsigned int* __restrict__ absmax_bits, BlockScalars* bs,
                                                         uint16_t* __restrict__ out) {
  constexpr int NS = SPLIT_FORMATS[PREC].pieces;
  PreScale ps{1.f, 1.f};
  if (PREC == PREC_FP16X2) ps = pre_scale(absmax >= 0.f ? absmax : __uint_as_float(*absmax_bits));
  if (blockIdx.x == 0 && threadIdx.x == 0 && !side_b) { bs->x_scale = ps.scale; bs->x_inv_scale = ps.inv; }
  const long long groups = Dp / 8, i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * groups) return;
  const long long n = i / groups;
  const int d = static_cast<int>(i - n * groups) * 8;
  const float* xr = x + n * D;
  float v[8];
  if (d + 7 < D && (D & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const float4 a4 = __ldg(reinterpret_cast<const float4*>(xr + d)), b4 = __ldg(reinterpret_cast<const float4*>(xr + d + 4));
    v[0] = a4.x; v[1] = a4.y; v[2] = a4.z; v[3] = a4.w; v[4] = b4.x; v[5] = b4.y; v[6] = b4.z; v[7] = b4.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = d + e < D ? __ldg(xr + d + e) : 0.f;
  }
  uint16_t p[8][3];
  uint4 pk[3];
  split8<PREC>(v, ps.scale, p, pk);
  store_kcat_row<PREC>(out + n * (mma_passes(NS) * Dp), Dp, d, pk, side_b);
}
void launch_eval_split(const float* x, int rows, int D, long long Dp, int prec, int side_b, float absmax, const unsigned int* absmax_bits,
                       BlockScalars* bs, uint16_t* out, cudaStream_t st) {
  const long long work = static_cast<long long>(rows) * (Dp / 8);
  with_prec(prec, [&](auto P) {
    eval_split_kernel<P><<<static_cast<unsigned int>((work + 255) / 256), 256, 0, st>>>(x, rows, D, Dp, side_b, absmax, absmax_bits, bs, out);
  });
  count_launch();
}

// Best positive of each query from the statistics sweep: max over same-label non-self gallery rows, -inf when there is none
__global__ void eval_best_kernel(RowArrays ra, int nq, float* __restrict__ best) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nq) best[i] = ra.cnt_same[i] > 0 ? ord2f(ra.st_maxw[i]) : -INFINITY;
}
void launch_eval_best(RowArrays ra, int nq, float* best, cudaStream_t st) {
  eval_best_kernel<<<(nq + 255) / 256, 256, 0, st>>>(ra, nq, best);
  count_launch();
}

// MAP@R: 64-bit segment offsets of the queries' positives, by one block.  Thread t sums a contiguous run of counts, the block scans
// the runs, and each thread writes its run's offsets.
__global__ void __launch_bounds__(1024) eval_seg_scan_kernel(const int* __restrict__ cnt, int nq, long long* __restrict__ seg, BlockScalars* bs,
                                                             unsigned long long* __restrict__ sum_err) {
  __shared__ long long s_warp[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int per = (nq + 1023) / 1024, i0 = min(nq, t * per), i1 = min(nq, i0 + per);
  long long run = 0;
  for (int i = i0; i < i1; ++i) run += cnt[i];
  long long incl = run;                                      // inclusive scan: across the warp, then across the warps
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) s_warp[w] = incl;
  __syncthreads();
  if (w == 0) {
    long long x = s_warp[lane], xi = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, xi, o);
      if (lane >= o) xi += y;
    }
    s_warp[lane] = xi - x;                                   // exclusive prefix of each warp
  }
  __syncthreads();
  long long off = s_warp[w] + incl - run;
  for (int i = i0; i < i1; ++i) { seg[i] = off; off += cnt[i]; }
  if (t == 1023) {
    seg[nq] = off;
    sum_err[0] = static_cast<unsigned long long>(off);
    sum_err[1] = static_cast<unsigned long long>(bs->err);
    bs->err = 0;
  }
}
void launch_eval_seg_scan(const int* cnt, int nq, long long* seg, BlockScalars* bs, unsigned long long* sum_err, cudaStream_t st) {
  eval_seg_scan_kernel<<<1, 1024, 0, st>>>(cnt, nq, seg, bs, sum_err);
  count_launch();
}

// One warp per query: the rank of each positive in its segment is the number of larger keys plus the number of equal keys before it,
// so every key lands on its own slot.  O(R_i^2 / 32) per query; the segments of metric-learning sets are short.
__global__ void __launch_bounds__(256) eval_seg_sort_kernel(const int* __restrict__ cnt, const long long* __restrict__ seg, int nq,
                                                            const float* __restrict__ src, float* __restrict__ dst) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= nq) return;
  const int R = cnt[i];
  const float* s = src + seg[i];
  float* d = dst + seg[i];
  for (int a = 0; a < R; a += 32) {
    const int k = a + lane;
    const uint32_t mine = k < R ? f2ord(s[k]) : 0u;
    int r = 0;
    for (int b = 0; b < R; b += 32) {
      const uint32_t other = b + lane < R ? f2ord(s[b + lane]) : 0u;
      const int n = min(32, R - b);
      for (int j = 0; j < n; ++j) {
        const uint32_t o = __shfl_sync(0xffffffffu, other, j);
        r += (o > mine || (o == mine && b + j < k)) ? 1 : 0;
      }
    }
    if (k < R) d[r] = ord2f(mine);
  }
}
void launch_eval_seg_sort(const int* cnt, const long long* seg, int nq, const float* src, float* dst, cudaStream_t st) {
  eval_seg_sort_kernel<<<(nq + 7) / 8, 256, 0, st>>>(cnt, seg, nq, src, dst);
  count_launch();
}

// One thread per query, k = 1..R ascending: neg_ge(k) = sum of hist[b < k], pos_k = k + neg_ge(k).  fp64, summed in ascending k and
// divided by R last, so a host loop in the same order gives the same bits.  rank = c_1 + neg_ge(1), c_1 = #{k : p_k = p_1}: the rank
// of npair_eval_rank.
__global__ void __launch_bounds__(256) eval_map_finish_kernel(const int* __restrict__ cnt, const long long* __restrict__ seg,
                                                              const int* __restrict__ fill, const float* __restrict__ pos,
                                                              const unsigned int* __restrict__ hist, int nq, double* __restrict__ map_r,
                                                              double* __restrict__ r_precision, int* __restrict__ R_out, int* __restrict__ rank) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const int R = cnt[i];
  double m = __longlong_as_double(0x7ff8000000000000ll), rp = m;
  int rk = 0;
  if (R > 0 && fill[i] == R) {
    const float* p = pos + seg[i];
    const unsigned int* h = hist + seg[i];
    int c1 = 1;
    while (c1 < R && p[c1] == p[0]) ++c1;
    rk = c1 + static_cast<int>(h[0]);
    double sum = 0.0;
    long long neg_ge = 0;
    int hits = 0;
    for (int k = 1; k <= R; ++k) {
      neg_ge += h[k - 1];
      const long long pk = k + neg_ge;
      if (pk > R) break;                                     // pos_k only grows with k
      sum += static_cast<double>(k) / static_cast<double>(pk);
      ++hits;
    }
    m = sum / R;
    rp = static_cast<double>(hits) / R;
  }
  map_r[i] = m;
  r_precision[i] = rp;
  if (R_out) R_out[i] = R;
  if (rank) rank[i] = rk;
}
void launch_eval_map_finish(const int* cnt, const long long* seg, const int* fill, const float* pos, const unsigned int* hist, int nq,
                            double* map_r, double* r_precision, int* R_out, int* rank, cudaStream_t st) {
  eval_map_finish_kernel<<<(nq + 255) / 256, 256, 0, st>>>(cnt, seg, fill, pos, hist, nq, map_r, r_precision, R_out, rank);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// k-means (npair_eval_kmeans, DESIGN 8.2): everything around the EPI_ARGMAX sweep
// --------------------------------------------------------------------------------------------
// Centroid c = row rows[c] of x.  Thread = one feature of one centroid.
__global__ void __launch_bounds__(256) km_gather_kernel(const float* __restrict__ x, int D, const int* __restrict__ rows, int k,
                                                        float* __restrict__ C) {
  const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<long long>(k) * D) return;
  const long long c = e / D;
  C[e] = x[static_cast<long long>(rows[c]) * D + (e - c * D)];
}
void launch_km_gather(const float* x, int D, const int* rows, int k, float* C, cudaStream_t st) {
  const long long work = static_cast<long long>(k) * D;
  km_gather_kernel<<<static_cast<unsigned int>((work + 255) / 256), 256, 0, st>>>(x, D, rows, k, C);
  count_launch();
}

// One warp per centroid: bias[c] = 0.5f * ||C_c||^2 in fp32 (per-lane fmaf chains over d = lane mod 32, then the warp tree), and the
// iteration's reset of counts[c]; thread 0 also clears the {changed, err, nonempty} words.
__global__ void __launch_bounds__(256) km_bias_kernel(const float* __restrict__ C, int k, int D, float* __restrict__ bias,
                                                      int* __restrict__ counts, KmeansWords* words) {
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) *words = KmeansWords{0u, 0u, 0u, 0u};
  if (c >= k) return;
  const float* r = C + static_cast<long long>(c) * D;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) s = fmaf(r[d], r[d], s);
  s = warp_sum(s);
  if (lane == 0) { bias[c] = 0.5f * s; counts[c] = 0; }
}
void launch_km_bias(const float* C, int k, int D, float* bias, int* counts, KmeansWords* words, cudaStream_t st) {
  km_bias_kernel<<<(k + 7) / 8, 256, 0, st>>>(C, k, D, bias, counts, words);
  count_launch();
}

// One warp per point: decode and clear its argmax key, count a changed assignment and a cluster's first member, and (accumulate)
// add the point's fixed-point features q = rint(x * sigma * 2^32) to its cluster's int64 sums.  Integer atomics: the sums do not
// depend on the order the points arrive in.
__global__ void __launch_bounds__(256) km_assign_kernel(unsigned long long* __restrict__ best, const float* __restrict__ x, int n, int D,
                                                        const unsigned int* __restrict__ absmax_bits, int k, int* __restrict__ assign,
                                                        int* __restrict__ counts, long long* __restrict__ sums, int accumulate,
                                                        KmeansWords* words) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  bool changed = false, first = false;
  if (i < n) {
    unsigned int a = 0;
    if (lane == 0) {
      const unsigned long long key = best[i];
      best[i] = 0;
      a = 0xFFFFFFFFu - static_cast<unsigned int>(key);
      if (key == 0 || a >= static_cast<unsigned int>(k)) { a = 0; atomicOr(&words->err, static_cast<unsigned int>(DERR_KMEANS_NO_ARGMAX)); }
      changed = assign[i] != static_cast<int>(a);
      assign[i] = static_cast<int>(a);
      first = atomicAdd(&counts[a], 1) == 0;
    }
    a = __shfl_sync(0xffffffffu, a, 0);
    if (accumulate) {
      const float sigma = pre_scale(__uint_as_float(*absmax_bits)).scale;
      const float* xr = x + static_cast<long long>(i) * D;
      unsigned long long* sr = reinterpret_cast<unsigned long long*>(sums + static_cast<long long>(a) * D);
      for (int d = lane; d < D; d += 32)    // x * sigma in (-1, 1) and the scaling by 2^32 are exact; one rounding, to nearest even
        atomicAdd(&sr[d], static_cast<unsigned long long>(__float2ll_rn((__ldg(xr + d) * sigma) * 4294967296.f)));
    }
  }
  const int n_changed = __syncthreads_count(changed), n_first = __syncthreads_count(first);
  if (threadIdx.x == 0) {
    if (n_changed) atomicAdd(&words->changed, static_cast<unsigned int>(n_changed));
    if (n_first) atomicAdd(&words->nonempty, static_cast<unsigned int>(n_first));
  }
}
void launch_km_assign(unsigned long long* best, const float* x, int n, int D, const unsigned int* absmax_bits, int k, int* assign,
                      int* counts, long long* sums, bool accumulate, KmeansWords* words, cudaStream_t st) {
  km_assign_kernel<<<(n + 7) / 8, 256, 0, st>>>(best, x, n, D, absmax_bits, k, assign, counts, sums, accumulate ? 1 : 0, words);
  count_launch();
}

// Thread = one feature of one centroid: the mean of a non-empty cluster, (float)(ldexp((double)sum / count, -32) * (1 / sigma)), every
// step exactly rounded so a host loop in fp64 gives the same bits; an empty cluster keeps its centroid.  Clears the sums.
__global__ void __launch_bounds__(256) km_update_kernel(long long* __restrict__ sums, const int* __restrict__ counts,
                                                        const unsigned int* __restrict__ absmax_bits, int k, int D, float* __restrict__ C) {
  const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= static_cast<long long>(k) * D) return;
  const int cnt = counts[e / D];
  if (cnt > 0) {
    const double inv = pre_scale(__uint_as_float(*absmax_bits)).inv;
    C[e] = static_cast<float>(ldexp(static_cast<double>(sums[e]) / static_cast<double>(cnt), -32) * inv);
    sums[e] = 0;
  }
}
void launch_km_update(long long* sums, const int* counts, const unsigned int* absmax_bits, int k, int D, float* C, cudaStream_t st) {
  const long long work = static_cast<long long>(k) * D;
  km_update_kernel<<<static_cast<unsigned int>((work + 255) / 256), 256, 0, st>>>(sums, counts, absmax_bits, k, D, C);
  count_launch();
}

// Inertia in fp64 in a fixed order: warp w of the fixed grid takes points w, w + KM_INERTIA_BLOCKS * 8, ..., each lane its features
// d = lane mod 32; the warp tree, the block's warps in order, then one thread over the blocks in order.
__global__ void __launch_bounds__(256) km_inertia_kernel(const float* __restrict__ x, const float* __restrict__ C,
                                                         const int* __restrict__ assign, int n, int D, double* __restrict__ partial) {
  __shared__ double s_w[8];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double s = 0.0;
  for (int i = blockIdx.x * 8 + w; i < n; i += KM_INERTIA_BLOCKS * 8) {
    const float* xr = x + static_cast<long long>(i) * D;
    const float* cr = C + static_cast<long long>(assign[i]) * D;
    for (int d = lane; d < D; d += 32) {
      const double e = static_cast<double>(xr[d]) - static_cast<double>(cr[d]);
      s = fma(e, e, s);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) s_w[w] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int j = 0; j < 8; ++j) b += s_w[j];
    partial[blockIdx.x] = b;
  }
}
__global__ void km_inertia_finish_kernel(const double* __restrict__ partial, double* __restrict__ out) {
  double s = 0.0;
  for (int b = 0; b < KM_INERTIA_BLOCKS; ++b) s += partial[b];
  *out = s;
}
void launch_km_inertia(const float* x, const float* C, const int* assign, int n, int D, double* partial, double* out, cudaStream_t st) {
  km_inertia_kernel<<<KM_INERTIA_BLOCKS, 256, 0, st>>>(x, C, assign, n, D, partial);
  km_inertia_finish_kernel<<<1, 1, 0, st>>>(partial, out);
  count_launch(2);
}

}  // namespace npair
