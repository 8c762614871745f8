// device.cuh -- device helpers that more than one kernel unit uses: the warp reductions, the operand split and the writer of the
// similarity GEMM's operands, and the reset of a row's statistics.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cfloat>

#include "kernels.cuh"

namespace npair {

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
// The packed pieces pk of features [d, d + 8) of row n into one side (side_b = false: A, true: B) of the similarity GEMM's operands,
// laid out by SimLayout.  Each piece is stored once; the GEMM forms the cross terms from the pieces in place (split_gemm_kernel).
template <int PREC>
__device__ __forceinline__ void store_sim_row(uint16_t* base, long long Dp, long long n, int d, const uint4 (&pk)[3], bool side_b) {
  constexpr int NS = SPLIT_FORMATS[PREC].pieces;
  const SimLayout L{NS, Dp};
#pragma unroll
  for (int s = 0; s < NS; ++s) *reinterpret_cast<uint4*>(base + L.offset(n, d, SimLayout::piece_slot(NS, s, side_b))) = pk[s];
}

// Row i's statistics before a similarity sweep accumulates into them (caffe_set of the stat blobs, .cu:230-236)
__device__ __forceinline__ void reset_row_stats(const RowArrays& ra, long long i) {
  ra.st_minw[i] = f2ord(FLT_MAX); ra.st_maxw[i] = f2ord(-FLT_MAX);
  ra.st_maxb[i] = f2ord(-FLT_MAX); ra.st_maxall[i] = f2ord(-FLT_MAX);
  ra.cnt_same[i] = 0;
}

}  // namespace npair
