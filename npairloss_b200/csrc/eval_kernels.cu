// eval_kernels.cu -- the retrieval evaluator's and k-means's kernels (DESIGN 8): operand preparation, the MAP@R segments and the
// k-means steps around the similarity GEMM's sweeps.
#include <cuda.h>
#include <cfloat>

#include "device.cuh"
#include "kernels.cuh"

namespace npair {

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

// Rows of x to one side of the similarity GEMM's operands (side_b = 0: the A side of the queries, 1: the B side of the gallery),
// through the layer's store_sim_row; rows [rows, round8(rows)) are zeros.  Thread = 8 features of one row.  With one piece consecutive
// threads walk a row; with two or three, eight consecutive threads take the 8 rows of a row group at the same features, so that their
// stores fill whole 128-byte core matrices.  The pre-scale is the layer's rule applied to max|x| over both sets: `absmax` when the
// caller gives it (>= 0), else *absmax_bits.
template <int PREC>
__global__ void __launch_bounds__(256) eval_split_kernel(const float* __restrict__ x, int rows, int D, long long Dp, int side_b, float absmax,
                                                         const unsigned int* __restrict__ absmax_bits, BlockScalars* bs,
                                                         uint16_t* __restrict__ out) {
  constexpr int NS = SPLIT_FORMATS[PREC].pieces;
  PreScale ps{1.f, 1.f};
  if (PREC == PREC_FP16X2) ps = pre_scale(absmax >= 0.f ? absmax : __uint_as_float(*absmax_bits));
  if (blockIdx.x == 0 && threadIdx.x == 0 && !side_b) { bs->x_scale = ps.scale; bs->x_inv_scale = ps.inv; }
  const long long groups = Dp / 8, i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= SimLayout{NS, Dp}.padded_rows(rows) * groups) return;
  long long n;
  int d;
  if (NS == 1) {
    n = i / groups; d = static_cast<int>(i - n * groups) * 8;
  } else {
    const long long gd = i >> 3, g = gd / groups;     // (row group, 8-feature chunk), row g * 8 + i % 8
    n = g * 8 + (i & 7); d = static_cast<int>(gd - g * groups) * 8;
  }
  const float* xr = x + n * D;
  float v[8];
  if (n >= rows) {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
  } else if (d + 7 < D && (D & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const float4 a4 = __ldg(reinterpret_cast<const float4*>(xr + d)), b4 = __ldg(reinterpret_cast<const float4*>(xr + d + 4));
    v[0] = a4.x; v[1] = a4.y; v[2] = a4.z; v[3] = a4.w; v[4] = b4.x; v[5] = b4.y; v[6] = b4.z; v[7] = b4.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = d + e < D ? __ldg(xr + d + e) : 0.f;
  }
  uint16_t p[8][3];
  uint4 pk[3];
  split8<PREC>(v, ps.scale, p, pk);
  store_sim_row<PREC>(out, Dp, n, d, pk, side_b);
}
void launch_eval_split(const float* x, int rows, int D, long long Dp, int prec, int side_b, float absmax, const unsigned int* absmax_bits,
                       BlockScalars* bs, uint16_t* out, cudaStream_t st) {
  const long long work = SimLayout{SPLIT_FORMATS[prec].pieces, Dp}.padded_rows(rows) * (Dp / 8);
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
      for (int d = lane; d < D; d += 32)    // x * sigma in (-2, 2) and the scaling by 2^32 are exact; one rounding, to nearest even
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

// --------------------------------------------------------------------------------------------
// k-means++ seeding (npair_eval_kmeans_seed, DESIGN 8.2): exact integer distances, so every sum is order-free and any grid gives the
// same bits.  Step t = the distance kernel (its last block picks the centre) + the update kernel (its last block draws step t + 1).
// --------------------------------------------------------------------------------------------
// u(seed, t, j): output number t * 256 + j + 1 of SplitMix64 seeded with `seed`
__device__ __forceinline__ unsigned long long kms_u(unsigned long long seed, int t, int j) {
  unsigned long long z = seed + (static_cast<unsigned long long>(t) * 256 + j + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Inclusive scan of one uint64 per thread over a block of KMS_THREADS threads; *total = the block's sum.  s_w: KMS_THREADS / 32 words.
__device__ unsigned long long kms_block_scan(unsigned long long v, unsigned long long* s_w, unsigned long long* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  __syncthreads();                                           // the previous scan has read s_w
  if (lane == 31) s_w[w] = incl;
  __syncthreads();
  unsigned long long before = 0, all = 0;
  for (int k = 0; k < KMS_THREADS / 32; ++k) {
    if (k < w) before += s_w[k];
    all += s_w[k];
  }
  *total = all;
  return before + incl;
}

// One warp per point: q = rint((x * sigma) * 2^13) (both products exact, one rounding to nearest even), rows padded with zeros to
// kms_dq(D); norm = sum q^2; dmin = UINT64_MAX (no centre yet).  Block 0 draws step 0's row.
__global__ void __launch_bounds__(256) kms_quantise_kernel(const float* __restrict__ x, int n, int D, const unsigned int* __restrict__ absmax_bits,
                                                           unsigned long long seed, int16_t* __restrict__ q, unsigned long long* __restrict__ norm,
                                                           unsigned long long* __restrict__ dmin, int* __restrict__ cand, KmSeedWords* words) {
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) cand[0] = static_cast<int>(__umul64hi(kms_u(seed, 0, 0), static_cast<unsigned long long>(n)));
  if (i >= n) return;
  // the points' pre-scale, halved where its clamped exponent leaves max|x * sigma| in [1, 2) (max|x| >= 2^127), so that |q| <= 2^13
  const float amax = __uint_as_float(*absmax_bits);
  const float sigma = pre_scale(amax).scale * (amax >= 0x1p127f ? 0.5f : 1.f);
  const long long Dq = kms_dq(D);
  const float* xr = x + static_cast<long long>(i) * D;
  int16_t* qr = q + i * Dq;
  unsigned long long s = 0;
  bool bad = false;
  for (int d = lane; d < Dq; d += 32) {
    const float v = d < D ? __ldg(xr + d) : 0.f;
    int qi = 0;
    if (isfinite(v)) qi = __float2int_rn((v * sigma) * 8192.f);
    else bad = true;
    qr[d] = static_cast<int16_t>(qi);
    s += static_cast<unsigned long long>(qi * qi);
  }
  s = warp_sum_u64(s);
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(&words->err, static_cast<unsigned int>(DERR_KMEANS_NO_ARGMAX));
  if (lane == 0) { norm[i] = s; dmin[i] = ~0ull; }
}
void launch_kms_quantise(const float* x, int n, int D, const unsigned int* absmax_bits, unsigned long long seed, int16_t* q,
                         unsigned long long* norm, unsigned long long* dmin, int* cand, KmSeedWords* words, cudaStream_t st) {
  kms_quantise_kernel<<<(n + 7) / 8, 256, 0, st>>>(x, n, D, absmax_bits, seed, q, norm, dmin, cand, words);
  count_launch();
}

// One thread per point.  The trials' rows are staged in shared memory as int32, KMS_LC trials by KMS_DC features at a time, and each
// thread reads its row 16 features (32 bytes) at a time: dot_j = sum q_i q_c in int32 per 16 features (|sum| <= 2^30), added in int64,
// and d(i, c) = ||q_i||^2 + ||q_c||^2 - 2 dot, exact.  Per-block sums of min(dmin, d) go to phi_acc by 64-bit integer atomics.
constexpr int KMS_LC = 16, KMS_DC = 512;
__global__ void __launch_bounds__(KMS_THREADS) kms_distance_kernel(const int16_t* __restrict__ q, const unsigned long long* __restrict__ norm,
                                                                   const unsigned long long* __restrict__ dmin, int n, int D,
                                                                   const int* __restrict__ cand, int L, int t,
                                                                   unsigned long long* __restrict__ dist, unsigned long long* phi_acc,
                                                                   int* __restrict__ rows, KmSeedWords* words) {
  __shared__ __align__(16) int s_c[KMS_LC][KMS_DC];
  __shared__ unsigned long long s_red[KMS_THREADS / 32][KMS_LC];
  __shared__ bool s_last;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int i = blockIdx.x * KMS_THREADS + tid;
  const bool live = i < n;
  const long long Dq = kms_dq(D);
  const int16_t* qr = q + static_cast<long long>(live ? i : 0) * Dq;
  const unsigned long long dm = live ? dmin[i] : 0, ni = live ? norm[i] : 0;
  for (int jc = 0; jc < L; jc += KMS_LC) {
    const int lc = min(KMS_LC, L - jc);
    long long acc[KMS_LC];
#pragma unroll
    for (int j = 0; j < KMS_LC; ++j) acc[j] = 0;
    for (long long d0 = 0; d0 < Dq; d0 += KMS_DC) {
      const int dc = static_cast<int>(min(static_cast<long long>(KMS_DC), Dq - d0));
      __syncthreads();                                       // every thread is done with the previous stage
      for (int e = tid; e < lc * dc; e += KMS_THREADS) {
        const int j = e / dc, d = e - j * dc;
        s_c[j][d] = q[static_cast<long long>(cand[jc + j]) * Dq + d0 + d];
      }
      __syncthreads();
      if (live) {
        for (int d = 0; d < dc; d += 16) {
          const int4 w0 = __ldg(reinterpret_cast<const int4*>(qr + d0 + d)), w1 = __ldg(reinterpret_cast<const int4*>(qr + d0 + d + 8));
          const int wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
          int a[16];
#pragma unroll
          for (int m = 0; m < 8; ++m) { a[2 * m] = static_cast<int16_t>(wv[m]); a[2 * m + 1] = wv[m] >> 16; }
#pragma unroll
          for (int j = 0; j < KMS_LC; ++j) {
            if (j < lc) {
              const int4* c4 = reinterpret_cast<const int4*>(&s_c[j][d]);
              int s = 0;
#pragma unroll
              for (int m = 0; m < 4; ++m) {
                const int4 c = c4[m];
                s += a[4 * m] * c.x + a[4 * m + 1] * c.y + a[4 * m + 2] * c.z + a[4 * m + 3] * c.w;
              }
              acc[j] += s;
            }
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < KMS_LC; ++j) {
      if (j < lc) {
        unsigned long long m = 0;
        if (live) {
          const unsigned long long dij = static_cast<unsigned long long>(static_cast<long long>(ni + norm[cand[jc + j]]) - 2 * acc[j]);
          dist[static_cast<long long>(jc + j) * n + i] = dij;
          m = dm < dij ? dm : dij;
        }
        m = warp_sum_u64(m);
        if (lane == 0) s_red[w][j] = m;
      }
    }
    __syncthreads();
    if (tid < lc) {
      unsigned long long s = 0;
      for (int k = 0; k < KMS_THREADS / 32; ++k) s += s_red[k][tid];
      atomicAdd(&phi_acc[jc + tid], s);
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(&words->ticket_dist, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last || tid != 0) return;
  __threadfence();
  unsigned long long best = 0;
  int jb = 0;
  for (int j = 0; j < L; ++j) {
    const unsigned long long v = atomicExch(&phi_acc[j], 0ull);   // read and clear for the next step
    if (j == 0 || v < best) { best = v; jb = j; }
  }
  words->jstar = static_cast<unsigned int>(jb);
  rows[t] = cand[jb];
  words->ticket_dist = 0;
}
void launch_kms_distance(const int16_t* q, const unsigned long long* norm, const unsigned long long* dmin, int n, int D, const int* cand,
                         int L, int t, unsigned long long* dist, unsigned long long* phi_acc, int* rows, KmSeedWords* words, cudaStream_t st) {
  kms_distance_kernel<<<(n + KMS_THREADS - 1) / KMS_THREADS, KMS_THREADS, 0, st>>>(q, norm, dmin, n, D, cand, L, t, dist, phi_acc, rows,
                                                                                   words);
  count_launch();
}

// One thread per point: dmin = min(dmin, d(i, centre t)), and the block's total.  The last block scans the totals into prefix (phi is
// the last), then per trial j of step t + 1: target = floor(u phi / 2^64), the block b whose inclusive prefix first exceeds it, and in b
// the first point whose inclusive prefix exceeds it (a point at distance 0 is never drawn); phi = 0 draws floor(u n / 2^64).
__global__ void __launch_bounds__(KMS_THREADS) kms_update_kernel(unsigned long long* __restrict__ dmin, const unsigned long long* __restrict__ dist,
                                                                 int n, unsigned long long seed, int t, int L_next,
                                                                 unsigned long long* __restrict__ totals, unsigned long long* __restrict__ prefix,
                                                                 int* __restrict__ cand, KmSeedWords* words) {
  __shared__ unsigned long long s_w[KMS_THREADS / 32];
  __shared__ bool s_last;
  const int tid = threadIdx.x, i = blockIdx.x * KMS_THREADS + tid;
  unsigned long long v = 0;
  if (i < n) {
    const unsigned long long dc = dist[static_cast<long long>(words->jstar) * n + i], d0 = dmin[i];
    v = dc < d0 ? dc : d0;
    dmin[i] = v;
  }
  unsigned long long tot;
  kms_block_scan(v, s_w, &tot);
  if (tid == 0) totals[blockIdx.x] = tot;
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(&words->ticket_upd, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int nb = gridDim.x;
  unsigned long long carry = 0;
  for (int b0 = 0; b0 < nb; b0 += KMS_THREADS) {
    const int b = b0 + tid;
    const unsigned long long incl = kms_block_scan(b < nb ? __ldcg(totals + b) : 0ull, s_w, &tot);
    if (b < nb) prefix[b] = carry + incl;
    carry += tot;
  }
  const unsigned long long phi = carry;
  if (tid == 0) { words->phi = phi; words->ticket_upd = 0; }
  __syncthreads();                                           // prefix is visible to the whole block
  for (int j = 0; j < L_next; ++j) {
    const unsigned long long u = kms_u(seed, t + 1, j);
    if (phi == 0) {
      if (tid == 0) cand[j] = static_cast<int>(__umul64hi(u, static_cast<unsigned long long>(n)));
      continue;
    }
    const unsigned long long target = __umul64hi(u, phi);    // < phi
    int lo = 0, hi = nb - 1;                                 // the first block with prefix > target
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (prefix[mid] > target) hi = mid; else lo = mid + 1;
    }
    const unsigned long long r = target - (lo ? prefix[lo - 1] : 0ull);
    const int idx = lo * KMS_THREADS + tid;
    const unsigned long long x = idx < n ? __ldcg(dmin + idx) : 0ull;
    const unsigned long long incl = kms_block_scan(x, s_w, &tot);
    if (incl > r && incl - x <= r) cand[j] = idx;
  }
}
void launch_kms_update(unsigned long long* dmin, const unsigned long long* dist, int n, unsigned long long seed, int t, int L_next,
                       unsigned long long* totals, unsigned long long* prefix, int* cand, KmSeedWords* words, cudaStream_t st) {
  kms_update_kernel<<<(n + KMS_THREADS - 1) / KMS_THREADS, KMS_THREADS, 0, st>>>(dmin, dist, n, seed, t, L_next, totals, prefix, cand, words);
  count_launch();
}

// --------------------------------------------------------------------------------------------
// hard negative class mining (npair_eval_class_batches, DESIGN 8.4): the greedy pick of each batch's classes from the stored S
// --------------------------------------------------------------------------------------------
// The maximum of a 64-bit key over the warp: of the high words, then of the low words among the lanes that hold the maximal high word
__device__ __forceinline__ unsigned long long warp_max_key(unsigned long long key) {
  const uint32_t hi = static_cast<uint32_t>(key >> 32), mh = __reduce_max_sync(0xffffffffu, hi);
  const uint32_t ml = __reduce_max_sync(0xffffffffu, hi == mh ? static_cast<uint32_t>(key) : 0u);
  return (static_cast<unsigned long long>(mh) << 32) | ml;
}

// One block of round_up(ceil(P / CB_ENTRIES), 32) threads per batch, as many as the SMs hold at once; the grid strides over the batches.
// Pool position j = tid + e * blockDim.x (e < CB_ENTRIES) lives in thread tid's registers: its
// class id[e] (-1 once picked, and past the pool) and v[e], the fmaxf of S over the picked classes' rows (NaN before the first term).
// A step gathers the last pick's row of S at every live id, all loads in flight together, folds them into v, and takes the block
// maximum of the distinct keys (ord(v) << 32) | ~j, ord(NaN) = 0, with 0 for a picked entry: a live key is never 0, since ~j has its
// top bits set.  Warp maxima, one shared-memory stage across the warps, and the winner's owner hands its class to every thread through
// shared memory: two barriers per step.  Keys are distinct, so the pick does not depend on the reduction order.
__global__ void __launch_bounds__(CB_THREADS) class_batch_kernel(const float* __restrict__ S, long long ldS, const int* __restrict__ pools,
                                                                 int P, int nb, int n, int* __restrict__ batches,
                                                                 float* __restrict__ scores) {
  __shared__ unsigned long long s_key[CB_THREADS / 32];
  __shared__ int s_pick;
  const int tid = threadIdx.x, lane = tid & 31, T = blockDim.x;
  const float qnan = __uint_as_float(0x7FC00000u);
  for (int t = blockIdx.x; t < nb; t += gridDim.x) {
    const int* pool = pools + static_cast<long long>(t) * P;
    int* out = batches + static_cast<long long>(t) * n;
    float* out_v = scores ? scores + static_cast<long long>(t) * n : nullptr;
    int id[CB_ENTRIES];
    float v[CB_ENTRIES];
#pragma unroll
    for (int e = 0; e < CB_ENTRIES; ++e) {
      const int j = tid + e * T;
      id[e] = j > 0 && j < P ? __ldg(pool + j) : -1;       // position 0, the seed, is picked
      v[e] = qnan;
    }
    int c = __ldg(pool);
    if (tid == 0) {
      out[0] = c;
      if (out_v) out_v[0] = qnan;
    }
    for (int s = 1; s < n; ++s) {
      const float* row = S + static_cast<long long>(c) * ldS;
      float x[CB_ENTRIES];
#pragma unroll
      for (int e = 0; e < CB_ENTRIES; ++e) x[e] = id[e] >= 0 ? __ldg(row + id[e]) : qnan;
      unsigned long long best = 0;
#pragma unroll
      for (int e = 0; e < CB_ENTRIES; ++e) {
        v[e] = fmaxf(v[e], x[e]);
        const unsigned long long key = (static_cast<unsigned long long>(v[e] != v[e] ? 0u : f2ord(v[e])) << 32) |
                                       static_cast<uint32_t>(~(tid + e * T));
        if (id[e] >= 0 && key > best) best = key;
      }
      best = warp_max_key(best);
      if (lane == 0) s_key[tid >> 5] = best;
      __syncthreads();
      best = warp_max_key(lane < (T >> 5) ? s_key[lane] : 0ull);
      const int win = static_cast<int>(~static_cast<uint32_t>(best));
      int picked = -1;
#pragma unroll
      for (int e = 0; e < CB_ENTRIES; ++e)
        if (tid + e * T == win) { picked = id[e]; id[e] = -1; }
      if (picked >= 0) {
        s_pick = picked;
        out[s] = picked;
        const uint32_t o = static_cast<uint32_t>(best >> 32);
        if (out_v) out_v[s] = o ? ord2f(o) : qnan;
      }
      __syncthreads();
      c = s_pick;
    }
  }
}
void launch_class_batches(const float* S, long long ldS, const int* pools, int P, int nb, int n, int* batches, float* scores, int sms,
                          cudaStream_t st) {
  static_assert(CB_THREADS * CB_ENTRIES >= CLASS_POOL_MAX, "one block holds the largest pool");
  const int threads = ((P + CB_ENTRIES - 1) / CB_ENTRIES + 31) / 32 * 32;
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, class_batch_kernel, threads, 0);
  const long long cap = static_cast<long long>(sms) * (per_sm > 0 ? per_sm : 1);
  class_batch_kernel<<<static_cast<int>(nb < cap ? nb : cap), threads, 0, st>>>(S, ldS, pools, P, nb, n, batches, scores);
  count_launch();
}

}  // namespace npair
