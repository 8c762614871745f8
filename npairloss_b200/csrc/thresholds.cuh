// thresholds.cuh -- the threshold pick of npair_multi_class_loss.cu:275-337 as device code.  The similarity GEMM's last CTA to finish
// runs it in place (one launch and ~10 us less per step); the SIMT backend's thresholds_kernel and, in world scope,
// thresholds_world_kernel (kernels.cu) share it.
#pragma once
#include <cfloat>
#include "kernels.cuh"

namespace npair {

// pos(SN,size) of npair_multi_class_loss.cu:285-287: size_t arithmetic for SN>=0, un-fused fp32 otherwise.
__device__ __forceinline__ bool pos_index(float sn, unsigned long long size, unsigned long long& pos) {
  if (size == 0) return false;
  if (sn >= 0.f) {                                    // -0.0f >= 0 is true
    const unsigned long long p = size - 1ull - static_cast<unsigned long long>(static_cast<long long>(static_cast<int>(sn)));
    if (p >= size) return false;
    pos = p; return true;
  }
  const float a = __ull2float_rn(size - 1ull);
  const float b = __fmul_rn(sn, __ull2float_rn(size));
  const float c = __fadd_rn(a, b);
  if (!(c > -2147483648.f && c < 2147483648.f)) return false;
  const int ip = static_cast<int>(c);                 // truncation toward zero
  if (ip < 0 || static_cast<unsigned long long>(ip) >= size) return false;
  pos = static_cast<unsigned long long>(ip); return true;
}
// The position of a relative select in its list of `size` entries; false with DERR_EMPTY_LIST (empty list) or DERR_POS_RANGE (SN puts
// the position outside the list) added to err
__device__ __forceinline__ bool side_position(unsigned long long size, float sn, unsigned long long& pos, int& err) {
  if (pos_index(sn, size, pos)) return true;
  err |= size == 0 ? DERR_EMPTY_LIST : DERR_POS_RANGE;
  return false;
}
__device__ __forceinline__ float clamp_thr(float v) { return v >= 0.f ? v : -FLT_MAX; }   // .cu:288,303,319,334

__host__ __device__ __forceinline__ bool is_rel(int m) { return m == M_RELATIVE_HARD || m == M_RELATIVE_EASY; }
__host__ __device__ inline bool sn_is_max(float sn) { return sn >= 0.f && static_cast<int>(sn) == 0; }   // pos = size-1

// The LOCAL-region thresholds of row i that are closed forms of its statistics (cs same-label pairs, min / max same-label and max
// diff-label similarity); a relative rule with any other SN is left to the radix select.  An empty list sets DERR_EMPTY_LIST in *err.
__device__ __forceinline__ void local_thresholds(const RowArrays& ra, const MiningParams& mp, int i, int N, int cs, float r_mn, float r_mxw,
                                                 float r_mxb, int* err) {
  if (mp.ap_region == REGION_LOCAL) {
    if (!is_rel(mp.ap_method)) ra.posi_thr[i] = r_mxb;                                                   // .cu:279
    else if (sn_is_max(mp.identsn)) { if (cs == 0) atomicOr(err, DERR_EMPTY_LIST); ra.posi_thr[i] = clamp_thr(r_mxw); }
  }
  if (mp.an_region == REGION_LOCAL) {
    if (!is_rel(mp.an_method)) ra.nega_thr[i] = r_mn;                                                    // .cu:310
    else if (sn_is_max(mp.diffsn)) { if (N - 1 - cs == 0) atomicOr(err, DERR_EMPTY_LIST); ra.nega_thr[i] = clamp_thr(r_mxb); }
  }
}

// The GLOBAL-region thresholds and the arming of the radix selects (.cu:292-337) from the statistics of `rows` rows of N columns: the
// reduction, in order from record 0, of n records `stride` floats apart (world scope: one per rank, rows = N; per rank: n = 1, rows = Q)
__device__ inline void finish_thresholds(const BlockStats* recs, int n, long long stride, unsigned long long rows, long long N,
                                         const MiningParams& mp, BlockScalars* bs) {
  BlockStats s = recs[0];
  for (int r = 1; r < n; ++r) {
    const BlockStats& t = rank_record(recs, stride, r);
    s.n_same += t.n_same; s.gmin_w = fminf(s.gmin_w, t.gmin_w); s.gmax_w = fmaxf(s.gmax_w, t.gmax_w); s.gmax_b = fmaxf(s.gmax_b, t.gmax_b);
    s.err |= t.err;
  }
  const unsigned long long n_same = s.n_same, n_diff = rows * static_cast<unsigned long long>(N - 1) - n_same;
  int err = s.err;
  float posi_g = 0.f, nega_g = 0.f;
  bool arm_ap = false, arm_an = false;
  if (mp.ap_region == REGION_GLOBAL) {
    if (!is_rel(mp.ap_method)) { if (n_diff == 0) err |= DERR_EMPTY_LIST; posi_g = s.gmax_b; }            // .cu:296
    else if (sn_is_max(mp.identsn)) { if (n_same == 0) err |= DERR_EMPTY_LIST; posi_g = clamp_thr(s.gmax_w); }   // pos = size-1
    else arm_ap = true;                                                                                    // .cu:300-304
  }
  if (mp.an_region == REGION_GLOBAL) {
    if (!is_rel(mp.an_method)) { if (n_same == 0) err |= DERR_EMPTY_LIST; nega_g = s.gmin_w; }             // .cu:327
    else if (sn_is_max(mp.diffsn)) { if (n_diff == 0) err |= DERR_EMPTY_LIST; nega_g = clamp_thr(s.gmax_b); }
    else arm_an = true;                                                                                    // .cu:331-335
  }
  bs->n_same = n_same; bs->n_diff = n_diff;
  bs->gmin_within = s.gmin_w; bs->gmax_within = s.gmax_w; bs->gmax_between = s.gmax_b;
  bs->posi_global = posi_g; bs->nega_global = nega_g;
  for (int side = 0; side < 2; ++side) {
    const bool arm = side == 0 ? arm_ap : arm_an;
    bs->sel_active[side] = 0;
    unsigned long long pos = 0;
    if (arm && side_position(side == 0 ? n_same : n_diff, side == 0 ? mp.identsn : mp.diffsn, pos, err)) {
      bs->sel_active[side] = 1; bs->sel_rank[side] = pos; bs->sel_prefix[side] = 0;
    }
  }
  bs->err |= err;
}

// Shared memory thresholds_one_block works in: 64-bit same-label counts and three extrema per warp, and the error word
constexpr int THRESHOLDS_SCRATCH_BYTES = 32 * 8 + 3 * 32 * 4 + 4;

// The threshold pick of Q rows by ONE block (any number of warps <= 32): LOCAL-region thresholds of every row, then the block's
// BlockStats, finished here (out == NULL) or written to *out (world scope: the rank's record for the exchange).  scratch:
// THRESHOLDS_SCRATCH_BYTES of 8-byte aligned shared memory.
__device__ inline void thresholds_one_block(RowArrays ra, int Q, int N, const MiningParams& mp, BlockScalars* bs, unsigned char* scratch,
                                            BlockStats* out) {
  unsigned long long* s_ns = reinterpret_cast<unsigned long long*>(scratch);          // [32]
  float* s_f = reinterpret_cast<float*>(scratch + 32 * 8);                            // [3][32]
  int* s_err = reinterpret_cast<int*>(scratch + 32 * 8 + 3 * 32 * 4);
  if (threadIdx.x == 0) *s_err = 0;
  __syncthreads();
  unsigned long long ns = 0; float mn = FLT_MAX, mxw = -FLT_MAX, mxb = -FLT_MAX;
  // U rows per thread and trip with all 4*U loads issued before the first use: the loop is a chain of L2 latencies otherwise
  // (measured: 15 us for 8192 rows on 384 threads with one row per trip)
  constexpr int U = 8;
  for (int i0 = threadIdx.x; i0 < Q; i0 += U * blockDim.x) {
    int cs_[U]; uint32_t a_[U], b_[U], c_[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * blockDim.x;
      if (i < Q) { cs_[u] = __ldcg(&ra.cnt_same[i]); a_[u] = __ldcg(&ra.st_minw[i]); b_[u] = __ldcg(&ra.st_maxw[i]); c_[u] = __ldcg(&ra.st_maxb[i]); }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * blockDim.x;
      if (i >= Q) break;
      const int cs = cs_[u];
      const float r_mn = ord2f(a_[u]), r_mxw = ord2f(b_[u]), r_mxb = ord2f(c_[u]);
      ns += static_cast<unsigned long long>(cs);
      mn = fminf(mn, r_mn); mxw = fmaxf(mxw, r_mxw); mxb = fmaxf(mxb, r_mxb);
      local_thresholds(ra, mp, i, N, cs, r_mn, r_mxw, r_mxb, s_err);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ns += __shfl_xor_sync(0xffffffffu, ns, o);
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mxw = fmaxf(mxw, __shfl_xor_sync(0xffffffffu, mxw, o)); mxb = fmaxf(mxb, __shfl_xor_sync(0xffffffffu, mxb, o));
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_ns[w] = ns; s_f[w] = mn; s_f[32 + w] = mxw; s_f[64 + w] = mxb; }
  __syncthreads();
  if (threadIdx.x == 0) {
    BlockStats s{0ull, FLT_MAX, -FLT_MAX, -FLT_MAX, *s_err};
    for (int k = 0; k < static_cast<int>(blockDim.x >> 5); ++k) {
      s.n_same += s_ns[k]; s.gmin_w = fminf(s.gmin_w, s_f[k]); s.gmax_w = fmaxf(s.gmax_w, s_f[32 + k]); s.gmax_b = fmaxf(s.gmax_b, s_f[64 + k]);
    }
    if (out) *out = s;
    else finish_thresholds(&s, 1, 0, static_cast<unsigned long long>(Q), N, mp, bs);
  }
}

}  // namespace npair
