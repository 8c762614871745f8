// kernels.cu -- HBM-bound kernels of the N-pair hot path (everything except the tensor-core contractions, gemm.cu, and the radix
// selects, select.cu).
// Each kernel cites the reference code it replaces (paths relative to /root/reference).
#include <cassert>
#include <cstdlib>
#include "device.cuh"
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
// abs_sum_max through 16-byte loads when x is 16-byte aligned (cudaMalloc'd / framework blobs are), 4-byte loads otherwise
__device__ __forceinline__ void abs_sum_max_at(const float* __restrict__ x, long long n, long long t0, long long stride, bool want_max,
                                               float& sum, float& mx) {
  if ((reinterpret_cast<uintptr_t>(x) & 15) == 0) abs_sum_max<true>(x, n, t0, stride, want_max, sum, mx);
  else abs_sum_max<false>(x, n, t0, stride, want_max, sum, mx);
}
// One kernel: per-block partial |x| sums (x_local) and max|x| (x_local and the database), the reset of the per-row statistics, and --
// in the last block to finish (ticket) -- the final asum, the power-of-two operand scale and the reset of the step state.
// The grid fixes the order of the asum: launch_prep_reduce sizes it from the larger of x_local and the database, so the asum of a
// memory step's current rows is summed in the order of one buffer of Q + m rows.  Eight blocks per SM cap it at 32 registers, which
// hold each sweep's four 16-byte loads in flight without spilling (uncapped, CUDA 12.9 allocates 40).
__global__ void __launch_bounds__(256, 8) prep_reduce_kernel(const float* __restrict__ xl, long long nl, RowSource db, int N, int D,
                                                             float* __restrict__ partial, int want_scale, RowArrays ra, int Q, BlockScalars* bs) {
  __shared__ float s_sum[8], s_max[8];
  __shared__ int s_last;
  float sum = 0.f, mx = 0.f;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  abs_sum_max_at(xl, nl, t0, stride, want_scale != 0, sum, mx);
  if (want_scale) {   // max |x| over the parts of the database that are not x_local itself (world 1: nothing more)
    const long long n0 = static_cast<long long>(db.n0) * D, n1 = static_cast<long long>(N) * D - n0;
    float unused = 0.f;
#pragma unroll 1
    for (int p = 0; p < 2; ++p) {
      const float* x = p ? db.x1 : db.x0;
      const long long n = p ? n1 : n0;
      if (n > 0 && (x != xl || n != nl)) abs_sum_max_at(x, n, t0, stride, true, unused, mx);
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
  if (!s_last) return;
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
}
// prep_reduce_kernel's two reductions for ring_prep_kernel, the same operations in the same order (prep_reduce_kernel keeps its own
// copy: calling these from it changes its register allocation).  The block totals: partial[block] = the block's sum and
// partial[1024 + block] its max; true in the last block to finish (ticket), which then finishes the step's prep in prep_finish
__device__ __forceinline__ bool prep_block_done(float sum, float mx, float* __restrict__ partial, BlockScalars* bs, float (&s_sum)[8],
                                                float (&s_max)[8]) {
  __shared__ int s_last;
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
  return s_last != 0;
}
// The last block: the asum and max |x| over the blocks' partials, the power-of-two operand scale and the reset of the step state
__device__ __forceinline__ void prep_finish(const float* __restrict__ partial, int want_scale, BlockScalars* bs, float (&s_max)[8]) {
  __threadfence();
  __shared__ double s_dsum[8];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  double dsum = 0.0; float mx = 0.f;
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
}
void launch_prep_reduce(const float* x_local, long long n_local, RowSource db, int N, int D, float* partial,
                        int want_scale, RowArrays ra, int Q, BlockScalars* bs, cudaStream_t st) {
  const long long n_total = static_cast<long long>(N) * D, nmax = n_local > n_total ? n_local : n_total;
  int nb = static_cast<int>((nmax + 256 * 16 - 1) / (256 * 16));
  if (nb < 1) nb = 1; if (nb > 592) nb = 592;
  prep_reduce_kernel<<<nb, 256, 0, st>>>(x_local, n_local, db, N, D, partial, want_scale, ra, Q, bs);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// operand split: the database's rows fp32 [N x D] -> Xs[s][N][ldXs] (K-major for the similarity GEMM) and the transposed
// XsT[s][D][ldXsT] (K-major for the gradient GEMM whose K is the sample index); XlT = local columns only.
// --------------------------------------------------------------------------------------------
// Block = 256 threads, tile = 32 rows (n) x 64 features (d).  Thread (nl = t/8, dg = t%8) converts 8 consecutive features of
// one row: two 16-byte loads, one 16-byte store per piece / section; the transposed pieces go through a shared tile so
// that they, too, are written as 16-byte row segments.
struct SplitArgs {
  RowSource x; int N, D;
  uint16_t* Xs; long long ldXs; uint16_t* XsT; long long ldXsT; uint16_t* XlT; long long ldXlT; int row0, Q;
  uint16_t *XcatA, *XcatB; long long Dp;
};
// The 8 features thread t of a block converts in tile (tile_d, tile_n).  Each row is loaded from its own buffer: a 32-row tile may
// straddle the two parts of a RowSource, and XsT is written in 16-byte segments of 8 rows, so a shifted pointer would not do.
__device__ __forceinline__ void split_load(const SplitArgs& a, int tile_d, int tile_n, float (&v)[8]) {
  const int N = a.N, D = a.D;
  const int t = threadIdx.x, nl = t >> 3, dg = t & 7;
  const int n = tile_n * 32 + nl, d = tile_d * 64 + 8 * dg;
  const bool rowok = n < N;
  const float* x = a.x.row(n, D);
  if (rowok && d + 7 < D && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {   // the row starts 16-byte aligned: so does x + d
    const float4 a4 = *reinterpret_cast<const float4*>(x + d);
    const float4 b4 = *reinterpret_cast<const float4*>(x + d + 4);
    v[0] = a4.x; v[1] = a4.y; v[2] = a4.z; v[3] = a4.w; v[4] = b4.x; v[5] = b4.y; v[6] = b4.z; v[7] = b4.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = (rowok && d + e < D) ? x[d + e] : 0.f;
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
  if (rowok && d < Dp && Xs) {     // Xs is NULL when the similarity GEMM reads the operands XcatA / XcatB below
    const long long ps = static_cast<long long>(N) * ldXs;
#pragma unroll
    for (int s = 0; s < NS; ++s) *reinterpret_cast<uint4*>(Xs + s * ps + static_cast<long long>(n) * ldXs + d) = pk[s];
  }
  // the similarity GEMM's operands (SimLayout): every row in the B format, and the rank's own rows, the only ones that are ever an A
  // operand, also in the A format at their local index; the rows that pad either side to a whole row group are zeros (v = 0 past N)
  if (PREC != PREC_BF16 && XcatA && d < Dp) {
    const SimLayout L{NS, Dp};
    if (n < L.padded_rows(N)) store_sim_row<PREC>(XcatB, Dp, n, d, pk, true);
    if (n >= row0 && n < row0 + L.padded_rows(Q)) {
      uint4 pa[3];
#pragma unroll
      for (int s = 0; s < 3; ++s) pa[s] = n < row0 + Q ? pk[s] : make_uint4(0u, 0u, 0u, 0u);
      store_sim_row<PREC>(XcatA, Dp, n - row0, d, pa, false);
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
// The labels of the Q current rows and the m memory rows into lab_total [Q + m], and the memory rows' records into rec[Q, Q + m): a
// memory row is never an anchor, so its record switches its transposed gradient term off exactly (RowRecord::memory) and keeps its label,
// which decides whether the anchor's own term treats the pair as same-label or different-label.
__global__ void memory_rows_kernel(const float* __restrict__ label, int Q, const float* __restrict__ mem_label, int m,
                                   float* __restrict__ lab_total, RowRecord* __restrict__ rec) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < Q + m; i += stride) {
    if (i < Q) { lab_total[i] = label[i]; continue; }
    const float l = mem_label[i - Q];
    lab_total[i] = l;
    rec[i] = RowRecord::memory(l);
  }
}
void launch_memory_rows(const float* label, int Q, const float* mem_label, int m, float* lab_total, RowRecord* rec, cudaStream_t st) {
  const int blocks = (Q + m + 255) / 256;
  memory_rows_kernel<<<blocks < 1024 ? blocks : 1024, 256, 0, st>>>(label, Q, mem_label, m, lab_total, rec);
  count_launch();
}

void launch_split(RowSource db, int N, int D, int prec, const BlockScalars* bs, uint16_t* Xs, long long ldXs,
                  uint16_t* XsT, long long ldXsT, uint16_t* XlT, long long ldXlT, int row0_local, int Q,
                  uint16_t* XcatA, uint16_t* XcatB, long long Dp, cudaStream_t st) {
  dim3 grid((D + 63) / 64, (N + 31) / 32);
  const SplitArgs a{db, N, D, Xs, ldXs, XsT, ldXsT, XlT, ldXlT, row0_local, Q, XcatA, XcatB, Dp};
  with_prec(prec, [&](auto P) { split_kernel<P><<<grid, 256, 0, st>>>(a, bs); });
  count_launch();
}

// --------------------------------------------------------------------------------------------
// cross-batch memory ring (npair_create_memory_ring, DESIGN 4.3.1)
// --------------------------------------------------------------------------------------------
// m = min(count, M), the memory rows a ring step over the device count would take
__device__ __forceinline__ int ring_rows(const Ring& r) {
  const unsigned long long c = r.st->count;
  return c < static_cast<unsigned long long>(r.M) ? static_cast<int>(c) : r.M;
}
// prep_reduce_kernel over [x; ring[0, m)] with the memory rows' max |x| taken from the slots' row maxima (a maximum has the same bits in
// any order, and each row maximum is the fmaxf of the same |x| values), on the grid launch_prep_reduce gives Q + m rows.  The last block
// then plans the step's refresh of the ring's operand pieces: the ring tiles [bt, nt) that split_tile must rewrite so that every
// piece equals what launch_split writes for this step's N = Q + m at this step's pre-scale.
__global__ void __launch_bounds__(256) ring_prep_kernel(const float* __restrict__ xl, int Q, int D, Ring r, int m, float* __restrict__ partial,
                                                        int want_scale, RowArrays ra, BlockScalars* bs) {
  __shared__ float s_sum[8], s_max[8];
  const bool bad = ring_rows(r) != m;
  float sum = 0.f, mx = 0.f;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  abs_sum_max_at(xl, static_cast<long long>(Q) * D, t0, stride, want_scale != 0, sum, mx);
  if (want_scale && !bad)
    for (long long i = t0; i < m; i += stride) mx = fmaxf(mx, __ldg(r.rowmax + i));
  for (long long i = t0; i < Q; i += stride) reset_row_stats(ra, i);
  if (!prep_block_done(sum, mx, partial, bs, s_sum, s_max)) return;
  prep_finish(partial, want_scale, bs, s_max);
  __syncthreads();
  RingState* rs = r.st;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  if (bad) {                                   // no slot is read, split or written this step
    if (t == 0) { rs->bad = 1; rs->n_list = 0; bs->err = DERR_RING_NOT_FULL; }
    return;
  }
  const float scale = *reinterpret_cast<volatile float*>(&bs->x_scale);
  const int bt = (Q + RING_TILE - 1) / RING_TILE, nt = (Q + m + RING_TILE - 1) / RING_TILE;
  const bool full = !rs->valid || rs->cached_scale != scale;
  const int boundary = m != rs->cached_m ? (Q + m - 1) / RING_TILE : -1;   // its rows past Q + m are zeros in the pieces
  __shared__ int s_cnt[8], s_base;
  if (t == 0) s_base = 0;
  for (int k0 = 0; k0 < nt; k0 += blockDim.x) {
    const int k = k0 + t;
    bool take = false;
    if (k < nt) {                              // every tile below nt is current after this step's split
      const int d = r.dirty[k];
      take = k >= bt && (full || d || k == boundary);
      if (d) r.dirty[k] = 0;
    }
    const unsigned int b = __ballot_sync(0xffffffffu, take);
    if (lane == 0) s_cnt[w] = __popc(b);
    __syncthreads();
    int off = s_base;
    for (int j = 0; j < w; ++j) off += s_cnt[j];
    if (take) r.list[off + __popc(b & ((1u << lane) - 1u))] = k;
    __syncthreads();
    if (t == 0) for (int j = 0; j < (blockDim.x >> 5); ++j) s_base += s_cnt[j];
    __syncthreads();
  }
  if (t == 0) { rs->n_list = s_base; rs->bad = 0; rs->valid = 1; rs->cached_m = m; rs->cached_scale = scale; }
}
void launch_ring_prep(const float* x, int Q, int D, Ring r, int m, float* partial, int want_scale, RowArrays ra, BlockScalars* bs,
                      cudaStream_t st) {
  const long long n_total = static_cast<long long>(Q + m) * D;    // launch_prep_reduce's grid for Q + m rows
  int nb = static_cast<int>((n_total + 256 * 16 - 1) / (256 * 16));
  if (nb < 1) nb = 1; if (nb > 592) nb = 592;
  ring_prep_kernel<<<nb, 256, 0, st>>>(x, Q, D, r, m, partial, want_scale, ra, bs);
  count_launch();
}

// The batch's tiles [0, bt), then the listed ring tiles, each split by split_load / split_tile as split_kernel splits it: a persistent
// grid, each block alternating its transposition buffers from tile to tile
template <int PREC>
__global__ void __launch_bounds__(256) ring_split_kernel(SplitArgs a, const BlockScalars* __restrict__ bs, const RingState* __restrict__ rs,
                                                         const int* __restrict__ list, int bt) {
  const int dt = (a.D + 63) / 64;
  const int total = (bt + rs->n_list) * dt;
  const float sc = (PREC == PREC_FP16X2) ? bs->x_scale : 1.f;
  int buf = 0;
  for (int i = blockIdx.x; i < total; i += gridDim.x, buf ^= 1) {
    const int k = i / dt, tile_d = i - k * dt;
    const int tile_n = k < bt ? k : __ldg(list + (k - bt));
    float v[8];
    split_load(a, tile_d, tile_n, v);
    split_tile<PREC>(a, sc, tile_d, tile_n, v, buf);
  }
}
void launch_ring_split(const float* x, int Q, int D, Ring r, int m, int prec, const BlockScalars* bs, uint16_t* Xs, long long ldXs,
                       uint16_t* XsT, long long ldXsT, uint16_t* XcatA, uint16_t* XcatB, long long Dp, int sms, cudaStream_t st) {
  const int N = Q + m, bt = (Q + RING_TILE - 1) / RING_TILE;
  const long long most = static_cast<long long>((N + RING_TILE - 1) / RING_TILE) * ((D + 63) / 64);
  const int grid = static_cast<int>(most < 8ll * sms ? most : 8ll * sms);
  const SplitArgs a{RowSource{x, Q, r.x}, N, D, Xs, ldXs, XsT, ldXsT, nullptr, 0, 0, Q, XcatA, XcatB, Dp};
  with_prec(prec, [&](auto P) { ring_split_kernel<P><<<grid, 256, 0, st>>>(a, bs, r.st, r.list, bt); });
  count_launch();
}

// One warp per pushed row: its D floats into the slot, max |x| of the row (fmaxf from 0, as abs_sum_max), the label and the tile's
// dirty flag; the last block advances the count
__global__ void __launch_bounds__(256) ring_push_kernel(const float* __restrict__ x, const float* __restrict__ label, int Q, int D, Ring r) {
  RingState* rs = r.st;
  if (rs->bad) return;
  const unsigned long long c = rs->count;
  const int M = r.M, lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5), gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  for (int row = (Q > M ? Q - M : 0) + gw; row < Q; row += warps) {   // a batch larger than the ring leaves its last M rows
    const int slot = static_cast<int>((c + static_cast<unsigned long long>(row)) % static_cast<unsigned long long>(M));
    const float* src = x + static_cast<long long>(row) * D;
    float* dst = r.x + static_cast<long long>(slot) * D;
    float mx = 0.f;
    for (int d = lane; d < D; d += 32) { const float v = src[d]; dst[d] = v; mx = fmaxf(mx, fabsf(v)); }
    mx = warp_max(mx);
    if (lane == 0) { r.rowmax[slot] = mx; r.label[slot] = label[row]; r.dirty[(Q + slot) / RING_TILE] = 1; }
  }
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) { __threadfence(); s_last = atomicAdd(&rs->ticket, 1u) == gridDim.x - 1; }
  __syncthreads();
  if (s_last && threadIdx.x == 0) { rs->count = c + static_cast<unsigned long long>(Q); rs->ticket = 0; }
}
void launch_ring_push(const float* x, const float* label, int Q, int D, Ring r, cudaStream_t st) {
  const int rows = Q < r.M ? Q : r.M;
  const int blocks = (rows + 7) / 8;
  ring_push_kernel<<<blocks < 1 ? 1 : (blocks > 1024 ? 1024 : blocks), 256, 0, st>>>(x, label, Q, D, r);
  count_launch();
}

__global__ void ring_tops_kernel(AsyncWords* __restrict__ aw, float* __restrict__ d_tops) {
  if (threadIdx.x != 0 || blockIdx.x != 0 || !(aw->tops.err & DERR_RING_NOT_FULL)) return;
  for (int t = 0; t < 5; ++t) d_tops[t] = __int_as_float(0x7fc00000);
  aw->err |= DERR_RING_NOT_FULL;
}
void launch_ring_tops(AsyncWords* aw, float* d_tops, cudaStream_t st) {
  ring_tops_kernel<<<1, 32, 0, st>>>(aw, d_tops);
  count_launch();
}

__global__ void __launch_bounds__(256) ring_loaded_kernel(Ring r, int m, int D, int tiles, unsigned long long count) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5), gw = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  for (int slot = gw; slot < m; slot += warps) {
    const float* src = r.x + static_cast<long long>(slot) * D;
    float mx = 0.f;
    for (int d = lane; d < D; d += 32) mx = fmaxf(mx, fabsf(src[d]));
    mx = warp_max(mx);
    if (lane == 0) r.rowmax[slot] = mx;
  }
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < tiles; k += gridDim.x * blockDim.x) r.dirty[k] = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    RingState* rs = r.st;
    rs->count = count; rs->valid = 0; rs->cached_m = 0; rs->cached_scale = 0.f; rs->bad = 0; rs->n_list = 0; rs->ticket = 0;
  }
}
void launch_ring_loaded(Ring r, int m, int D, int tiles, unsigned long long count, cudaStream_t st) {
  const int blocks = (m + 7) / 8;
  ring_loaded_kernel<<<blocks < 1 ? 1 : (blocks > 1024 ? 1024 : blocks), 256, 0, st>>>(r, m, D, tiles, count);
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
// same size gives the same bits.  anchor_w (or NULL): the loss sums the fp32 products w_i log(A_i / T_i) (0 at w_i = 0) in the same
// order; at w = 1 they are the unweighted terms, bit for bit.
__device__ __forceinline__ void lse_finalize_block(int Q, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* __restrict__ tops,
                                                   TopSums* __restrict__ xout, unsigned int seq, const float* __restrict__ anchor_w) {
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
      if (anchor_w) {                                           // a masked row adds 0, even where its log is -inf (A / T underflowed)
        const float wv = ok ? __ldg(&anchor_w[r]) : 0.f;
        lv[u] = wv == 0.f ? 0.f : lv[u] * wv;
      }
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
    // err through L2: the row pass's blocks set DERR_ANCHOR_WEIGHT during this launch, and this block's L1 may hold the line
    TopSums s{0.0, {0, 0, 0}, bs->asum, __ldcg(&bs->err)};
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
                                                       int num_tops, TopsBlock* __restrict__ tops,
                                                       float m2c_off /*log2(world) - k*/, float wscale /*2^k: weight_scale_log2*/,
                                                       TopSums* __restrict__ xout /*world scope: this rank's tops sums, else NULL*/,
                                                       int wpr /*warps per row: 1, 2, 4 or 8 (few rows per rank: keep the SMs full)*/,
                                                       unsigned int seq /*written behind the tops: the host polls it*/, int finalize,
                                                       const float* __restrict__ anchor_w /*[Q] or NULL*/, float* __restrict__ row_loss /*[Q] or NULL*/) {
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
      const float lv = (A == 0.f || T == 0.f) ? 0.f : logf(A / T);  // .cu:162-169
      ra.logv[i] = lv;
      if (row_loss) row_loss[i] = -lv;                          // the unweighted per-anchor loss (DESIGN 4.5)
      const int lim = N - 2;
      ra.hits[i] = (cs > 0 && c <= min(1, lim)) ? 1 : 0;
      ra.hits[Q + i] = (cs > 0 && c <= min(5, lim)) ? 1 : 0;
      ra.hits[2 * Q + i] = (cs > 0 && c <= min(10, lim)) ? 1 : 0;
      const float invA = A == 0.f ? 0.f : 1.f / A;              // Get_Query_Diff_Part zero rules (.cu:410-415)
      const float invT = T == 0.f ? 0.f : 1.f / T;
      const float cA = invT - invA;
      // The factors 2^k / A and 2^k / T overflow for sums below about 2^(k - 128) (selected positives ~79 nats below the row maximum
      // at k = 14).  Such a row moves 2^j of its factors into its exponent offset: the builders' exponential 2^(s log2(e) - (m2 - j))
      // is e 2^j <= 2^j, the factors are 2^(k - j) / A, and every weight e 2^j * 2^(k - j) (1/T - 1/A) keeps its value in
      // [-2^k, 2^k].  j = max(0, k - 127 - floor(log2 A)) <= k - 1 (a nonzero A is a sum of normal terms, >= 2^-126) leaves every
      // factor below 2^127; rows with j = 0 keep every bit.  m2c carries no j: it is only an exponent offset of 2^k e / T / world.
      const float amin = A > 0.f ? A : T;
      const int j = amin > 0.f ? max(0, ilogbf(wscale) - 127 - ilogbf(amin)) : 0;
      const float fsc = ldexpf(wscale, -j);
      // The anchor weight w (DESIGN 4.5) scales every term of the row: the factors by w, and the diff-label weight, which lives in the
      // exponent offset m2c, by 2^-log2(w) (+inf at w = 0).  Exact at w = 1 and at w = 2^-i; without weights w = 1.
      float m2c = T == 0.f ? INFINITY : m2 + log2f(T) + m2c_off;
      float w = 1.f;
      if (anchor_w) {
        w = __ldg(&anchor_w[i]);
        if (!(w >= 0.f && w <= 1.f)) atomicOr(&bs->err, DERR_ANCHOR_WEIGHT);
        m2c = w > 0.f ? m2c - log2f(w) : INFINITY;
      }
      ra.rowrec[i] = RowRecord::make(m2c, thr_n, m2 - static_cast<float>(j), li, thr_p, cA * fsc * w, invT * fsc * w);
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
  lse_finalize_block(Q, ra, bs, num_tops, tops, xout, seq, anchor_w);
}
__global__ void lse_finalize_kernel(int Q, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* __restrict__ tops, unsigned int seq,
                                    const float* __restrict__ anchor_w) {
  lse_finalize_block(Q, ra, bs, num_tops, tops, nullptr, seq, anchor_w);
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
                     int wlog2, unsigned int seq, bool finalize, AnchorIO aio, cudaStream_t st) {
  int wpr = 1, threads = 256;
  lse_shape(sim.Q, sim.N, &wpr, &threads);
  const int rows_per_blk = threads / 32 / wpr;
  const int grid = (sim.rows + rows_per_blk - 1) / rows_per_blk;
  const float log2_world = xout ? 0.f : log2f(static_cast<float>(world));
  lse_rows_kernel<<<grid, threads, 0, st>>>(sim, mp, ra, bs, num_tops, tops_dev, log2_world - static_cast<float>(wlog2), ldexpf(1.f, wlog2), xout,
                                            wpr, seq, finalize ? 1 : 0, aio.weight, aio.row_loss);
  count_launch();
}
void launch_lse_finalize(int Q, int N, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* tops_dev, unsigned int seq, const float* anchor_w,
                         cudaStream_t st) {
  int wpr = 1, threads = 256;
  lse_shape(Q, N, &wpr, &threads);
  lse_finalize_kernel<<<1, threads, 0, st>>>(Q, ra, bs, num_tops, tops_dev, seq, anchor_w);
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
// MODE BW_ROWSCAL (world > 1): the similarity GEMM is bitwise symmetric ACROSS ranks (role-symmetric instructions), so the
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
// Range: the fast path is one pass over the row with no scaling.  When its sum of squares ss is not in [L2_SS_MIN, FLT_MAX] (the
// squares overflowed, or so many of them were subnormal that their rounding could show), the row is redone on x 2^-e, e the
// exponent of max|x| clamped as in pre_scale: the scaling is exact, so y is the fast path's y of the scaled row, and 1/||x|| is that
// row's 1/||x|| times 2^-e (+inf above FLT_MAX).  A row the fast path accepts gives the bits it gave before the rescue existed.
// A row with a NaN or +-inf element gives a NaN row and a NaN 1/||x||; an all-zero row gives zeros.
// --------------------------------------------------------------------------------------------
// ss >= 2^-64: the fast path rounds at most D partial sums in the subnormal range, 2^-150 each, i.e. at most D 2^-86 of ss
constexpr float L2_SS_MIN = 0x1p-64f;
// the sum of the squares of x * sc in the order every pass uses; sc = 1 (SCALED false) on the fast path
template <bool SCALED>
__device__ __forceinline__ float l2norm_row_ss(const float* xr, int dim, int lane, bool vec, bool quad, float sc) {
  auto f = [sc](float v) { return SCALED ? v * sc : v; };
  float ss = 0.f;
  if (vec) for (int d = lane * 4; d < dim; d += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + d);
    const float a = f(v.x), b = f(v.y), c = f(v.z), e = f(v.w);
    ss = fmaf(a, a, ss); ss = fmaf(b, b, ss); ss = fmaf(c, c, ss); ss = fmaf(e, e, ss);
  } else if (quad) for (int d = lane * 4; d < dim; d += 128) for (int e = 0; e < 4; ++e) { const float a = f(xr[d + e]); ss = fmaf(a, a, ss); }
  else for (int d = lane; d < dim; d += 32) { const float a = f(xr[d]); ss = fmaf(a, a, ss); }
  return warp_sum(ss);
}
template <bool SCALED>
__device__ __forceinline__ void l2norm_row_store(const float* xr, float* yr, int dim, int lane, bool vec, float sc, float nrm) {
  auto f = [sc](float v) { return SCALED ? v * sc : v; };
  if (vec) for (int d = lane * 4; d < dim; d += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + d);
    *reinterpret_cast<float4*>(yr + d) = make_float4(f(v.x) / nrm, f(v.y) / nrm, f(v.z) / nrm, f(v.w) / nrm);
  } else for (int d = lane; d < dim; d += 32) yr[d] = f(xr[d]) / nrm;
}
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
  const float ss = l2norm_row_ss<false>(xr, dim, lane, vec, quad, 1.f);   // the same value in every lane: the branch is warp-uniform
  float inv;
  if (ss >= L2_SS_MIN && ss <= FLT_MAX) {
    const float nrm = sqrtf(ss);
    inv = 1.f / nrm;
    l2norm_row_store<false>(xr, yr, dim, lane, vec, 1.f, nrm);
  } else {
    float mx = 0.f;                                                     // fmaxf skips a NaN; ss has caught it
    for (int d = lane; d < dim; d += 32) mx = fmaxf(mx, fabsf(xr[d]));
    mx = warp_max(mx);
    const bool nonfinite = ss != ss || !(mx <= FLT_MAX);               // a NaN or +-inf element
    if (nonfinite || mx == 0.f) {                                       // ... or a zero row
      const float fill = nonfinite ? __int_as_float(0x7fc00000) : 0.f;
      inv = fill;
      for (int d = lane; d < dim; d += 32) yr[d] = fill;
    } else {
      const PreScale ps = pre_scale(mx);
      const float nrm = sqrtf(l2norm_row_ss<true>(xr, dim, lane, vec, quad, ps.scale));
      inv = (1.f / nrm) * ps.scale;
      l2norm_row_store<true>(xr, yr, dim, lane, vec, ps.scale, nrm);
    }
  }
  if (lane == 0 && inv_norm) inv_norm[r] = inv;
}
// t * inv, except that t = 0 stays 0 where inv = +inf (a row with 1/||x|| above FLT_MAX): such a row's gradient is +-inf or 0.  A
// finite inv gives the bits of t * inv either way, and a NaN inv a NaN.
__device__ __forceinline__ float l2norm_dx(float t, float inv) { return t == 0.f && inv == INFINITY ? t : t * inv; }
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
    *reinterpret_cast<float4*>(dr + d) = make_float4(l2norm_dx(g.x - a.x * dot, inv), l2norm_dx(g.y - a.y * dot, inv),
                                                     l2norm_dx(g.z - a.z * dot, inv), l2norm_dx(g.w - a.w * dot, inv));
  } else for (int d = lane; d < dim; d += 32) dr[d] = l2norm_dx(gr[d] - yr[d] * dot, inv);
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

__global__ void async_tops_kernel(AsyncWords* __restrict__ aw, int num_tops, float* __restrict__ d_tops) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int err = aw->tops.err & (DERR_EMPTY_LIST | DERR_POS_RANGE | DERR_ANCHOR_WEIGHT);
  for (int t = 0; t < 5; ++t) d_tops[t] = err ? __int_as_float(0x7fc00000) : (t < num_tops ? aw->tops.tops[t] : 0.f);
  aw->err |= static_cast<unsigned int>(err);
}
void launch_async_tops(AsyncWords* aw, int num_tops, float* d_tops, cudaStream_t st) {
  async_tops_kernel<<<1, 32, 0, st>>>(aw, num_tops, d_tops);
  count_launch();
}
// The fp32 operations of backward_core's host alpha (lw_over_q, then 0.5f times it) and of the GEMMs' alpha * *dev_scale, in order:
// IEEE division and multiplications (no fast math), and an exact ldexpf
__global__ void grad_scale_kernel(const float* __restrict__ d_lw, int Q, int wlog2, const BlockScalars* __restrict__ bs,
                                  AsyncWords* __restrict__ aw) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float lw_over_q = ldexpf(__fdiv_rn(*d_lw, static_cast<float>(Q)), -wlog2);
  aw->grad_scale = __fmul_rn(__fmul_rn(0.5f, lw_over_q), bs->x_inv_scale);
}
void launch_grad_scale(const float* d_lw, int Q, int wlog2, const BlockScalars* bs, AsyncWords* aw, cudaStream_t st) {
  grad_scale_kernel<<<1, 32, 0, st>>>(d_lw, Q, wlog2, bs, aw);
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

}  // namespace npair
