// kernels.cuh -- device-side data structures shared by the memory-bound kernels and the host context.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace npair {

// mining enums: caffe.proto:8-18
enum { REGION_GLOBAL = 0, REGION_LOCAL = 1 };
enum { M_HARD = 0, M_EASY = 1, M_RAND = 2, M_RELATIVE_HARD = 3, M_RELATIVE_EASY = 4 };

// device error bits (the reference has undefined behaviour in these cases: SURVEY.md 9.4 Q5)
enum { DERR_EMPTY_LIST = 1, DERR_POS_RANGE = 2 };

// operand split formats (see gemm_wgmma.cuh)
enum { PREC_BF16X3 = 0, PREC_BF16 = 1, PREC_FP16X2 = 2 };

// Global (per-rank-block) scalars living in device memory.
struct BlockScalars {
  unsigned long long n_same, n_diff;       // sizes of ident_global / diff_global (.cu:225-265)
  float gmin_within, gmax_within;          // min / max over all same-label pairs of the block
  float gmax_between;                      // max over all diff-label pairs (diff_global.back(), .cu:296)
  float posi_global, nega_global;          // GLOBAL-region thresholds (valid when the region is GLOBAL)
  int err;                                 // DERR_* bits
  unsigned int ticket;                     // block-completion counter of the row pass (last block finalises)
  unsigned int ticket2;                    // block-completion counter of the thresholds kernel
  unsigned int ticket0;                    // block-completion counter of the prep kernel
  // radix-select state, one per side (0 = AP over same pairs, 1 = AN over diff pairs)
  unsigned long long sel_rank[2];          // remaining 0-based rank inside the current prefix bucket
  uint32_t sel_prefix[2];                  // ordered-uint prefix decided so far
  uint32_t sel_mask[2];                    // which bits of the prefix are decided
  int sel_active[2];                       // 1 while a GLOBAL relative select is in flight
  unsigned long long sel_cnt[2];           // population of the chosen first-digit bucket (GLOBAL select)
  unsigned int cand_n[2];                  // entries of the compact candidate lists (GLOBAL select)
  unsigned int ticket3;                    // block-completion counter of the GLOBAL select kernels
  float asum;                              // sum |x| over the local features (.cu:400)
  float x_absmax;                          // max |x| over x_total (operand pre-scale for PREC_FP16X2)
  float x_scale, x_inv_scale;              // power of two s.t. max|x*scale| in [0.5,1]; 1 for other precisions
};

struct MiningParams {
  int ap_region, ap_method, an_region, an_method;
  float margin_ident, margin_diff, identsn, diffsn;
};

struct RowArrays {
  // statistics written by the sim-GEMM epilogue (ordered-uint encoded)
  uint32_t *st_minw, *st_maxw, *st_maxb, *st_maxall;
  int* cnt_same;
  // thresholds WITHOUT margin (posi_thr / nega_thr of .cu:275-337)
  float *posi_thr, *nega_thr;
  // forward row results
  float *A, *T, *logv;
  int* hits;                 // [3][Q] retrieval hit flags for k=1,5,10
  // row scalars consumed by the backward: [Q][8] floats {m2c, thr_n', max_all*log2e, label | thr_p', cA, cT, 0} (see lse_rows_kernel)
  // (one 32-byte record per row: all-gathered as is when world > 1, bulk-copied per K block by the fused gradient kernel)
  float* rowscal;
};

// order-preserving float <-> uint32 map so atomicMin/atomicMax work on floats of either sign
__host__ __device__ __forceinline__ uint32_t f2ord(float f) {
#ifdef __CUDA_ARCH__
  uint32_t b = __float_as_uint(f);
#else
  union { float f; uint32_t u; } c; c.f = f; uint32_t b = c.u;
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(uint32_t u) {
  uint32_t b = (u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  union { float f; uint32_t u; } c; c.u = b; return c.f;
#endif
}

// Number of kernels this library has launched in this process (every launch site bumps it; read through
// npair_kernel_launches(): bench.py reports the per-step delta as gpu_launches).
extern unsigned long long g_kernel_launches;
inline void count_launch(int n = 1) { g_kernel_launches += static_cast<unsigned long long>(n); }

// launchers (kernels.cu)
void launch_absmax_asum(const float* x_local, long long n_local, const float* x_total, long long n_total,
                        float* partial /*[2*1024]*/, BlockScalars* bs, int want_scale, cudaStream_t st);
void launch_prep_reduce(const float* x_local, long long n_local, const float* x_total, long long n_total, float* partial /*[2*1024]*/,
                        int want_scale, RowArrays ra, int Q, BlockScalars* bs, cudaStream_t st);
void launch_split(const float* x_total, int N, int D, int prec, const BlockScalars* bs,
                  uint16_t* Xs, long long ldXs /*Dp*/, uint16_t* XsT, long long ldXsT /*Np*/,
                  uint16_t* XlT, long long ldXlT /*Qp, or 0*/, int row0_local, int Q,
                  uint16_t* XcatA /*or NULL*/, uint16_t* XcatB, long long Dp, cudaStream_t st);
void launch_row_stats_ref(const float* S, long long ldS, int Q, int N, const float* lab_rows, const float* lab_cols,
                          int self_offset, RowArrays ra, cudaStream_t st);
// xout: NULL, or (world scope) 6 floats receiving this rank's block statistics instead of the final thresholds
void launch_thresholds(RowArrays ra, int Q, int N, MiningParams mp, BlockScalars* bs, float* scratch /*>= 2 KB*/, float* xout, cudaStream_t st);
void launch_thresholds_world(const float* xall, int xstride, int world, long long N, MiningParams mp, BlockScalars* bs, cudaStream_t st);
void launch_tops_world(const float* xall, int xstride, int world, long long N, int num_tops, float* tops_dev, unsigned int seq, cudaStream_t st);
// side_mask: bit 0 = AP threshold over the same-label list, bit 1 = AN threshold over the diff-label list
void launch_local_select(const float* S, long long ldS, int Q, int N, const float* lab_rows, const float* lab_cols,
                         int self_offset, int side_mask, float sn_ap, float sn_an, RowArrays ra, BlockScalars* bs, int sms, bool force_warp_kernel, cudaStream_t st);
// lets the current device launch the one-warp-per-row local select with its dynamic shared memory (above the default limit)
cudaError_t allow_local_select_smem();
void launch_global_select_pass(const float* S, long long ldS, int Q, int N, const float* lab_rows, const float* lab_cols,
                               int self_offset, int side_mask, int pass /*0,1,2*/, RowArrays ra, unsigned long long* hist /*[2][2048], zero*/,
                               uint32_t* cand /*[2][cand_cap]*/, unsigned int cand_cap, int world_scope, BlockScalars* bs, int sms, cudaStream_t st);
// world scope: xall = the ranks' exchanged [2][2048] 64-bit digit counts
void launch_global_decide(const float* xall, int xstride, int world, int side_mask, int pass, RowArrays ra, int Q, unsigned long long* hist,
                          uint32_t* cand, unsigned int cand_cap, BlockScalars* bs, cudaStream_t st);
// Row pass over rows [row0, row0 + rows) of the rank (S points at row row0's similarities; lab_rows, self_offset and ra are the
// rank's).  finalize: the last block also reduces the Q rows' results into the tops; otherwise launch_lse_finalize does, once.
void launch_lse_rows(const float* S, long long ldS, int Q, int N, const float* lab_rows, const float* lab_cols,
                     int self_offset, MiningParams mp, RowArrays ra, BlockScalars* bs, int num_tops, float* tops_dev /*[5]+err*/,
                     int world, float* xout /*world scope: 7 floats of partial tops, else NULL*/, unsigned int seq, int row0, int rows,
                     bool finalize, cudaStream_t st);
void launch_lse_finalize(int Q, int N, RowArrays ra, BlockScalars* bs, int num_tops, float* tops_dev, unsigned int seq, cudaStream_t st);
// mode: BW_SPLIT (world > 1, reduce-scatter form: H and HT), BW_SYM (world == 1), BW_ROWSCAL (world > 1, row-scalar
// exchange: rs_total = all-gathered [world][5][Q] row scalars)
enum { BW_SPLIT = 0, BW_SYM = 1, BW_ROWSCAL = 2 };
void launch_build_weights(const float* S, long long ldS, int Q, int N, const float* lab_rows, const float* lab_cols,
                          int self_offset, int world, int mode, const float* rs_total, MiningParams mp, RowArrays ra, int prec,
                          uint16_t* H, long long ldH /*Np*/, uint16_t* HT, long long ldHT /*Qp*/, cudaStream_t st);
void launch_l2norm_fwd(const float* x, int rows, int dim, float* y, float* inv_norm, cudaStream_t st);
void launch_l2norm_bwd(const float* y, const float* inv_norm, const float* dy, int rows, int dim, float* dx, cudaStream_t st);

}  // namespace npair
