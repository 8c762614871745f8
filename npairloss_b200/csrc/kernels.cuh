// kernels.cuh -- device-side data structures shared by the memory-bound kernels and the host context.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <cmath>
#include <type_traits>

namespace npair {

// mining enums: caffe.proto:8-18
enum { REGION_GLOBAL = 0, REGION_LOCAL = 1 };
enum { M_HARD = 0, M_EASY = 1, M_RAND = 2, M_RELATIVE_HARD = 3, M_RELATIVE_EASY = 4 };

// device error bits (the reference has undefined behaviour in these cases: SURVEY.md 9.4 Q5)
enum { DERR_EMPTY_LIST = 1, DERR_POS_RANGE = 2 };
// retrieval evaluation: the MAP@R gather found more positives in a row than the statistics sweep counted
enum { DERR_GATHER_SLOT = 4 };
// k-means: a point's assignment sweep found no column with a score above -inf (a NaN or infinite input)
enum { DERR_KMEANS_NO_ARGMAX = 8 };
// the layer: an anchor weight (npair_set_anchor_io) outside [0, 1] or NaN
enum { DERR_ANCHOR_WEIGHT = 16 };
// a ring forward (npair_forward_ring) found fewer rows in the context's memory ring than the m it was enqueued for: a replayed graph
// after npair_memory_ring_load with count < M
enum { DERR_RING_NOT_FULL = 32 };

constexpr float LOG2E = 1.4426950408889634f;

// Operand split formats (gemm_wgmma.cuh): an fp32 value is stored as `pieces` 2-byte pieces whose sum reproduces it.
enum { PREC_BF16X3 = 0, PREC_BF16 = 1, PREC_FP16X2 = 2 };
struct SplitFormat {
  int pieces;   // 2-byte pieces per value, largest first
  bool bf16;    // element type of the pieces: bf16, else fp16
};
constexpr SplitFormat SPLIT_FORMATS[3] = {{3, true} /*PREC_BF16X3*/, {1, true} /*PREC_BF16*/, {2, false} /*PREC_FP16X2*/};
// MMA passes of a product of two operands of `pieces` pieces: one per piece pair (a, b) with a + b < pieces, in the order of
// pass_pieces.
__host__ __device__ constexpr int mma_passes(int pieces) { return pieces * (pieces + 1) / 2; }

// The operands of the bitwise-symmetric similarity GEMM (DESIGN 5), one A-side and one B-side buffer of `rows` rows of Dp features.
//   pieces == 1 (bf16): plain rows [rows][Dp], read in 64-element K blocks through a 128B-swizzled map.
//   pieces >= 2: every piece once, in wgmma's no-swizzle core-matrix order.  A row group g = n / 8 holds, per K block kb of BK
//     features, one 16*BK-byte block per piece slot: BK / 8 core matrices of 8 rows x 8 features (128 contiguous bytes each):
//       element (n, k) of slot s at  ((g * Dp / BK + kb) * pieces + s) * 8 * BK + (k % BK) / 8 * 64 + (n % 8) * 8 + k % 8
//     so one TMA box {8 * BK, pieces, 1 K block, row groups} is a run of 16 * BK * pieces contiguous bytes per row group.  The slot of
//     a piece differs between the sides (piece_slot): a cross-term instruction takes core matrix 0 from one piece and core matrix 1
//     from another piece at the same features, through the descriptor's leading byte offset, which has to be positive.
//     Rows [rows, round8(rows)) are zeros.
struct SimLayout {
  int pieces;
  long long Dp;     // a multiple of 64
  __host__ __device__ constexpr static int bk_of(int pieces) { return pieces == 1 ? 64 : (pieces == 2 ? 32 : 16); }
  __host__ __device__ int bk() const { return bk_of(pieces); }
  __host__ __device__ long long padded_rows(long long rows) const { return pieces == 1 ? rows : (rows + 7) / 8 * 8; }
  __host__ __device__ long long elems(long long rows) const { return padded_rows(rows) * pieces * Dp; }
  // slot of piece s (0 = largest) in side A: the pieces in order; in side B: the largest piece last (fp16x2 [lo][hi], bf16x3
  // [mid][lo][hi]), so that every cross term (hi, x) has core matrix 1 behind core matrix 0 on both sides
  __host__ __device__ static int piece_slot(int pieces, int s, bool side_b) { return side_b ? (s == 0 ? pieces - 1 : s - 1) : s; }
  // element offset of feature k (a multiple of 8) of row n, piece slot `slot`
  __host__ __device__ long long offset(long long n, long long k, int slot) const {
    if (pieces == 1) return n * Dp + k;
    const int bk = bk_of(pieces);
    return (((n >> 3) * (Dp / bk) + k / bk) * pieces + slot) * 8 * bk + (k % bk) / 8 * 64 + (n & 7) * 8;
  }
};
// Calls f(std::integral_constant<int, PREC>()) for the runtime format `prec`: where a kernel instantiation is chosen by format.
template <class F>
inline decltype(auto) with_prec(int prec, F&& f) {
  if (prec == PREC_BF16) return f(std::integral_constant<int, PREC_BF16>());
  if (prec == PREC_FP16X2) return f(std::integral_constant<int, PREC_FP16X2>());
  return f(std::integral_constant<int, PREC_BF16X3>());
}

// Every selection rule of .cu:79-120 is rewritten as ONE compare  sgn*s <= thr'  with a per-row transformed threshold:
//   s <  t  <=>   s <= nextbelow(t)         s <= t  <=>   s <= t
//   s >= t  <=>  -s <= -t                   s >  t  <=>  -s <= nextbelow(-t)          ALL  <=>  s <= +inf
// (exact for every float incl. +-0 and the -FLT_MAX / FLT_MAX sentinels; NaN compares false on both sides).
__host__ __device__ __forceinline__ float ap_sign(int m) { return (m == M_EASY || m == M_RELATIVE_EASY) ? -1.f : 1.f; }
__host__ __device__ __forceinline__ float an_sign(int m) { return (m == M_HARD || m == M_RELATIVE_HARD) ? -1.f : 1.f; }
__device__ __forceinline__ float ap_thr(float t, int m) {     // same-label rule on t = posi_thr + margin_ident
  switch (m) {
    case M_HARD: return nextafterf(t, -INFINITY);            // s <  t
    case M_EASY: return -t;                                  // s >= t
    case M_RAND: return INFINITY;
    case M_RELATIVE_HARD: return t;                          // s <= t
    default: return -t;                                      // RELATIVE_EASY: s >= t
  }
}
__device__ __forceinline__ float an_thr(float t, int m) {     // diff-label rule on t = nega_thr + margin_diff
  switch (m) {
    case M_HARD: return nextafterf(-t, -INFINITY);           // s >  t
    case M_EASY: return t;                                   // s <= t
    case M_RAND: return INFINITY;
    case M_RELATIVE_HARD: return -t;                         // s >= t
    default: return t;                                       // RELATIVE_EASY: s <= t
  }
}

// What the backward needs of one row, written by the forward row pass (lse_rows_kernel).  It crosses GPUs as raw bytes (peer-memory
// pushes, the NCCL all-gather, npair_row_scalars / npair_backward_gathered), so this is the one description of its layout.  The two
// 16-byte halves are loaded and stored as vectors; the first holds all that a diff-label pair needs.
//   m2     max_all * log2(e) - j, the row's exponent offset
//   m2c    max_all * log2(e) + log2(T) + log2(world) - k (+inf when T == 0): a diff-label weight 2^k exp(s - max) / T / world is ONE
//          exponential 2^(s*log2(e) - m2c)
//   thr_n  the an_thr-transformed diff-label threshold;  thr_p  the ap_thr-transformed same-label threshold
//   cA     same-label weight factor 2^(k-j) (1/T - 1/A);  cT  diff-label weight factor 2^(k-j) / T
// so every gradient weight built from records, 2^(s*log2(e) - m2) times a factor, comes out scaled by 2^k, k = weight_scale_log2(format),
// and the gradient GEMM's alpha carries 2^-k.  j is 0 except on rows whose 2^k / A or 2^k / T could pass 2^127 (lse_rows_kernel).
// A weighted anchor (npair_set_anchor_io, DESIGN 4.5) carries its weight w in [0, 1] in the record: cA w, cT w, and m2c - log2(w)
// (+inf at w = 0), so every term of the row, its own and its transposed ones, comes out scaled by w.  At w = 1 these are the bits above.
struct RowRecord {
  float4 lo, hi;   // {m2c, thr_n, m2, label}, {thr_p, cA, cT, 0}
  __host__ __device__ static RowRecord make(float m2c, float thr_n, float m2, float label, float thr_p, float cA, float cT) {
    return RowRecord{make_float4(m2c, thr_n, m2, label), make_float4(thr_p, cA, cT, 0.f)};
  }
  // records[k] addressed in 16-byte halves (the gradient kernel's shared-memory reads are scheduled for this address arithmetic)
  __host__ __device__ static RowRecord load(const RowRecord* records, int k) {
    const float4* h = reinterpret_cast<const float4*>(records);
    return RowRecord{h[2 * k], h[2 * k + 1]};
  }
  // The record of a cross-batch memory row (DESIGN 4.3), which is never an anchor: +inf exponent offsets, -inf thresholds and zero
  // weight factors make its transposed gradient term exactly 0 in both weight builders; its label is the row's real one, since the
  // anchor's own term tells same-label from different-label pairs by the column record's label
  __host__ __device__ static RowRecord memory(float label) { return make(INFINITY, -INFINITY, INFINITY, label, -INFINITY, 0.f, 0.f); }
  __host__ __device__ float m2c() const { return lo.x; }
  __host__ __device__ float thr_n() const { return lo.y; }
  __host__ __device__ float m2() const { return lo.z; }
  __host__ __device__ float label() const { return lo.w; }
  __host__ __device__ float thr_p() const { return hi.x; }
  __host__ __device__ float cA() const { return hi.y; }
  __host__ __device__ float cT() const { return hi.z; }
};
static_assert(sizeof(RowRecord) == 32, "row records are exchanged as 32 raw bytes");
// log2 of the scale the gradient weights of format `prec` are built at.  An fp16x2 weight is split into fp16 hi + lo pieces; unscaled,
// the lo piece of a weight below about 2^-3 falls into fp16's subnormal range (spacing 2^-24), an absolute error of up to 2^-25 per
// weight, which does not average out when the rows are clustered and their weights nearly equal.  Every weight lies in [-1, 1]
// (exp(s - max) / T and exp(s - max) (1/T - 1/A) with exp(s - max) <= A <= T; the factors 1/A and 1/T alone do not, and the row
// record's exponent offset absorbs what of 2^k / A would overflow, RowRecord), and the world-1 operand H = g'(j, m) + g'(m, j) in
// [-2, 2]; 2^14 * 2 = 32768 stays below fp16's largest finite 65504 (2^15 * 2 would not), so k = 14 is the largest safe scale and
// keeps the lo piece normal down to weights of about 2^-17.  bf16 pieces have fp32's exponent range: no scale.
__host__ __device__ constexpr int weight_scale_log2(int prec) { return prec == PREC_FP16X2 ? 14 : 0; }
constexpr long long ROW_RECORD_FLOATS = sizeof(RowRecord) / sizeof(float);   // exchanges count floats

// One rank's contribution to a world-scope reduction (global_scope), exchanged as raw bytes in its slot of the small exchange; the
// per-rank finish is the same reduction over the one record of its own rank.
// The statistics the threshold pick reduces over a block of rows (finish_thresholds, thresholds.cuh): the number of same-label pairs,
// min / max same-label and max diff-label similarity, DERR_* bits
struct BlockStats {
  unsigned long long n_same;
  float gmin_w, gmax_w, gmax_b;
  int err;
};
static_assert(sizeof(BlockStats) == 24, "block statistics are exchanged as 24 raw bytes");
// The sums the tops are made of (publish_tops, kernels.cu): sum of the rows' log(A/T), retrieval hits at k = 1, 5, 10, sum |x|, DERR_* bits
struct TopSums {
  double loss_sum;
  int hits[3];
  float asum;
  int err;
};
static_assert(sizeof(TopSums) == 32, "tops sums are exchanged as 32 raw bytes");
// Record r of an exchange that holds one record per rank, `stride` floats apart
template <class T>
__host__ __device__ __forceinline__ const T& rank_record(const T* recs, long long stride, int r) {
  return *reinterpret_cast<const T*>(reinterpret_cast<const float*>(recs) + r * stride);
}

// What a forward publishes to the host, in mapped pinned memory: the tops, the DERR_* bits, then the forward's sequence number, which
// is stored last (the host polls it)
struct TopsBlock {
  float tops[5];
  int err;
  unsigned int seq;
};

// The asynchronous step's words in device memory (npair_forward_async, npair_backward_device_weight; DESIGN 4.4): the forward publishes
// its tops here instead of to the host, the error bits of its forwards gather until npair_async_status, and a backward's gradient
// scale is computed here from the device loss weight
struct AsyncWords {
  TopsBlock tops;
  unsigned int err;        // DERR_* bits of the asynchronous forwards since the last status call
  float grad_scale;        // (1/2)(lw/Q) 2^-k times the operand's inverse pre-scale: the gradient GEMMs' alpha * *dev_scale
};

// Global (per-rank-block) scalars living in device memory.
struct BlockScalars {
  unsigned long long n_same, n_diff;       // sizes of ident_global / diff_global (.cu:225-265)
  float gmin_within, gmax_within;          // min / max over all same-label pairs of the block
  float gmax_between;                      // max over all diff-label pairs (diff_global.back(), .cu:296)
  float posi_global, nega_global;          // GLOBAL-region thresholds (valid when the region is GLOBAL)
  int err;                                 // DERR_* bits
  unsigned int ticket;                     // block-completion counter of the row pass (last block finalises)
  unsigned int ticket2;                    // block-completion counter of the similarity sweep (its last CTA picks the thresholds)
  unsigned int ticket0;                    // block-completion counter of the prep kernel
  // radix-select state, one per side (0 = AP over same pairs, 1 = AN over diff pairs)
  unsigned long long sel_rank[2];          // remaining 0-based rank inside the current prefix bucket
  uint32_t sel_prefix[2];                  // ordered-uint prefix decided so far
  uint32_t reserved_[2];                   // unused; holds the fields below at their offsets (moved 8 bytes down, x_absmax .. x_inv_scale
                                           // share the first 128-byte line with the tickets, and the B=8192 D=512 step measured ~1 % slower
                                           // on an H100 80GB HBM3 at 700 W)
  int sel_active[2];                       // 1 while a GLOBAL relative select is in flight
  unsigned long long sel_cnt[2];           // population of the chosen first-digit bucket (GLOBAL select)
  unsigned int cand_n[2];                  // entries of the compact candidate lists (GLOBAL select)
  unsigned int ticket3;                    // block-completion counter of the GLOBAL select kernels
  float asum;                              // sum |x| over the local features (.cu:400)
  float x_absmax;                          // max |x| over x_total (operand pre-scale for PREC_FP16X2)
  float x_scale, x_inv_scale;              // pre_scale(x_absmax) for PREC_FP16X2; 1 for other precisions
};

// The operand pre-scale of a set whose largest |x| is `absmax`: scale = 2^-e and inv = 2^e, with absmax = m 2^e, m in [0.5, 1), and e
// clamped to [-126, 127] so that both are finite (at e = 127 the scale is the subnormal 2^-127, exact since nothing here is built with
// -ftz).  max|x * scale| is in [0.5, 1) for absmax in [2^-127, 2^127), below 0.5 under it and in [1, 2) above it; the scaling is exact
// either way, and the inverse undoes it exactly.  1 when absmax is 0 or not finite.
struct PreScale { float scale, inv; };
__host__ __device__ inline PreScale pre_scale(float absmax) {
  float sc = 1.f, inv = 1.f;
  if (absmax > 0.f && isfinite(absmax)) {
    int e; frexpf(absmax, &e);                 // absmax = m * 2^e, m in [0.5,1)
    e = e < -126 ? -126 : (e > 127 ? 127 : e);
    sc = ldexpf(1.f, -e); inv = ldexpf(1.f, e);
  }
  return PreScale{sc, inv};
}

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
  RowRecord* rowrec;         // [Q] what the backward needs of each row
};

// What one launch reads of the rank's Q x N similarity matrix: rows [row0, row0 + rows) of the rank, which the buffer S holds from
// its row 0 (a materialised S is the one block row0 = 0, rows = Q).  Kernels index RANK rows i -- labels, RowArrays (hits[k * Q + i]
// included) -- unshifted and reach row i's similarities through row(i).  Row i's self pair is column self_col(i), excluded by
// position whatever its label (a NaN label equals nothing, its own included).  Kernels take the view as a const __grid_constant__
// parameter (a plain one spills more in the selects, CUDA 12.9); its pointers are no __restrict__ parameters, so loads that must
// stay read-only say so with __ldg.
struct SimRows {
  const float* S;
  long long ldS;
  int Q, N;                  // the rank's rows, the world's columns
  int row0, rows;
  const float* lab_rows;     // [Q] the rank's labels
  const float* lab_cols;     // [N] the world's labels
  int col0;                  // world column of rank row 0: rank * Q
  __host__ __device__ __forceinline__ const float* row(int i) const { return S + static_cast<long long>(i - row0) * ldS; }
  __host__ __device__ __forceinline__ int self_col(int i) const { return i + col0; }
  // whether row i's self column is one of the four columns j4 .. j4 + 3
  __host__ __device__ __forceinline__ bool self_in4(int i, int j4) const { return !(self_col(i) < j4 || self_col(i) > j4 + 3); }
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

// The database's N rows of D features, in at most two buffers: rows [0, n0) from x0, rows [n0, N) from x1 at row n - n0.  One buffer:
// n0 = N, x1 = NULL.  A cross-batch memory step (DESIGN 4.3) reads [x; x_mem] as {x, Q, x_mem}, where the rows lie.
struct RowSource {
  const float* x0; int n0; const float* x1 = nullptr;
  __host__ __device__ __forceinline__ const float* row(int n, int D) const {
    return n < n0 ? x0 + static_cast<long long>(n) * D : x1 + static_cast<long long>(n - n0) * D;
  }
};

// launchers (kernels.cu)
// The step's operand preparation: sum |x| over the n_local elements of x_local (the top asum), and when want_scale, max |x| over
// x_local and the N x D database `db` (the pre-scale); also resets the Q rows' statistics and the step state in bs
void launch_prep_reduce(const float* x_local, long long n_local, RowSource db, int N, int D, float* partial /*[2*1024]*/,
                        int want_scale, RowArrays ra, int Q, BlockScalars* bs, cudaStream_t st);
void launch_split(RowSource db, int N, int D, int prec, const BlockScalars* bs,
                  uint16_t* Xs, long long ldXs /*Dp*/, uint16_t* XsT, long long ldXsT /*Np*/,
                  uint16_t* XlT, long long ldXlT /*Qp, or 0*/, int row0_local, int Q,
                  uint16_t* XcatA /*or NULL*/, uint16_t* XcatB, long long Dp, cudaStream_t st);
// lab_total[0, Q + m) = [label; mem_label], rec[Q + i] = RowRecord::memory(mem_label[i])
void launch_memory_rows(const float* label, int Q, const float* mem_label, int m, float* lab_total, RowRecord* rec, cudaStream_t st);

// The cross-batch memory ring a context keeps (npair_create_memory_ring, DESIGN 4.3.1).  Slot s holds a row the layer used and its
// label; it is database row Q + s of a step with m = min(count, M) memory rows.  The split operand pieces of the ring's rows stay in
// the context's operand buffers from step to step: a step re-splits only the 32-row database tiles (RING_TILE) whose pieces are stale.
constexpr int RING_TILE = 32;                   // the rows of one split_tile
struct RingState {
  unsigned long long count;    // rows pushed since the last load
  int valid;                   // the pieces of rows [Q, Q + cached_m) were split at the pre-scale cached_scale
  int cached_m;
  float cached_scale;
  int bad;                     // this step's m is not min(count, M): nothing reads or writes the slots (DERR_RING_NOT_FULL)
  int n_list;                  // ring tiles this step re-splits: list[0, n_list)
  unsigned int ticket;         // last-block counter of the push
};
struct Ring {
  float *x, *label, *rowmax;   // [M][D] rows, [M] labels, [M] max |x| of each slot's row
  int* dirty;                  // [database tiles] 1: a slot of the tile was pushed since its pieces were split
  int* list;                   // [database tiles] the ring tiles the step re-splits, ascending
  RingState* st;
  int M;
};
// A ring step's launches, in order.  prep: launch_prep_reduce over [x; ring[0, m)] (same grid, asum bits and x_absmax), with max |x|
// of the memory rows from the slots' row maxima; its last block also flags a step whose m is not min(count, M) and lists the ring
// tiles to re-split: all of them when the pre-scale differs from the cached one, else those with a pushed slot and, when m changed,
// the tile of row Q + m - 1.
void launch_ring_prep(const float* x, int Q, int D, Ring r, int m, float* partial, int want_scale, RowArrays ra, BlockScalars* bs,
                      cudaStream_t st);
// split: writes what launch_split writes for [x; ring[0, m)], for the Q batch rows' tiles and the listed ring tiles only
void launch_ring_split(const float* x, int Q, int D, Ring r, int m, int prec, const BlockScalars* bs, uint16_t* Xs, long long ldXs,
                       uint16_t* XsT, long long ldXsT, uint16_t* XcatA, uint16_t* XcatB, long long Dp, int sms, cudaStream_t st);
// push: the last min(Q, M) rows of x and their labels into slots (count + r) mod M, their row maxima, the tiles' dirty flags, count += Q
void launch_ring_push(const float* x, const float* label, int Q, int D, Ring r, cudaStream_t st);
// the asynchronous forward's finish after launch_async_tops: NaN tops and the error bit kept in aw->err for a DERR_RING_NOT_FULL step
void launch_ring_tops(AsyncWords* aw, float* d_tops, cudaStream_t st);
// after a load of m = min(count, M) slots: their row maxima, the count, no valid pieces, no dirty tile
void launch_ring_loaded(Ring r, int m, int D, int tiles, unsigned long long count, cudaStream_t st);
void launch_row_stats_ref(SimRows sim, RowArrays ra, cudaStream_t st);
// The threshold pick of the rank's Q rows by one block (SIMT backend; the tensor-core similarity sweep runs it in its last CTA)
void launch_thresholds(RowArrays ra, int Q, int N, MiningParams mp, BlockScalars* bs, cudaStream_t st);
// World scope: the thresholds of the world's N rows from the ranks' BlockStats, which lie xstride floats apart in xall
void launch_thresholds_world(const float* xall, int xstride, int world, long long N, MiningParams mp, BlockScalars* bs, cudaStream_t st);
// World scope: the tops of the world's N rows from the ranks' TopSums, which lie xstride floats apart in xall
void launch_tops_world(const float* xall, int xstride, int world, long long N, int num_tops, TopsBlock* tops_dev, unsigned int seq, cudaStream_t st);
// Row pass over the rows of sim.  finalize: the last block also reduces the Q rows' results into the tops; otherwise
// launch_lse_finalize does, once.  xout: NULL, or (world scope) receives the rank's TopSums instead of the tops.  wlog2: the records'
// weight scale, weight_scale_log2 of the operand format.  AnchorIO: the rank's Q anchor weights and per-anchor loss output (DESIGN 4.5),
// each NULL when unused
struct AnchorIO { const float* weight; float* row_loss; };
void launch_lse_rows(SimRows sim, MiningParams mp, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* tops_dev, int world, TopSums* xout,
                     int wlog2, unsigned int seq, bool finalize, AnchorIO aio, cudaStream_t st);
void launch_lse_finalize(int Q, int N, RowArrays ra, BlockScalars* bs, int num_tops, TopsBlock* tops_dev, unsigned int seq, const float* anchor_w,
                         cudaStream_t st);
// mode: BW_SPLIT (world > 1, reduce-scatter form: H and HT), BW_SYM (world == 1), BW_ROWSCAL (rs_total = one record per column: at
// world > 1 the world's N row records, all-gathered; in a cross-batch memory step at world 1, the Q row records followed by the m
// memory rows' RowRecord::memory records, whose transposed terms are 0)
enum { BW_SPLIT = 0, BW_SYM = 1, BW_ROWSCAL = 2 };
// over the rank's whole S (sim.row0 == 0, sim.rows == Q)
void launch_build_weights(SimRows sim, int world, int mode, const RowRecord* rs_total, MiningParams mp, RowArrays ra, int prec,
                          uint16_t* H, long long ldH /*Np*/, uint16_t* HT, long long ldHT /*Qp*/, cudaStream_t st);
// The asynchronous forward's finish: d_tops[0, 5) = what the host would read of aw->tops (0 past num_tops), or NaN with the error bits
// added to aw->err when a DERR_EMPTY_LIST / DERR_POS_RANGE / DERR_ANCHOR_WEIGHT bit is set
void launch_async_tops(AsyncWords* aw, int num_tops, float* d_tops, cudaStream_t st);
// aw->grad_scale = (0.5f * ldexpf(*d_lw / Q, -wlog2)) * bs->x_inv_scale: the host's alpha of the gradient GEMMs times their device scale,
// in the same fp32 operations
void launch_grad_scale(const float* d_lw, int Q, int wlog2, const BlockScalars* bs, AsyncWords* aw, cudaStream_t st);
void launch_l2norm_fwd(const float* x, int rows, int dim, float* y, float* inv_norm, cudaStream_t st);
void launch_l2norm_bwd(const float* y, const float* inv_norm, const float* dy, int rows, int dim, float* dx, cudaStream_t st);

// launchers of the radix selects (select.cu)
// side_mask: bit 0 = AP threshold over the same-label list, bit 1 = AN threshold over the diff-label list
void launch_local_select(SimRows sim, int side_mask, float sn_ap, float sn_an, RowArrays ra, BlockScalars* bs, int sms, bool force_warp_kernel, cudaStream_t st);
// lets the current device launch the one-warp-per-row local select with its dynamic shared memory (above the default limit)
cudaError_t allow_local_select_smem();
// over the rank's whole S (sim.row0 == 0, sim.rows == Q)
void launch_global_select_pass(SimRows sim, int side_mask, int pass /*0,1,2*/, RowArrays ra, unsigned long long* hist /*[2][2048], zero*/,
                               uint32_t* cand /*[2][cand_cap]*/, unsigned int cand_cap, int world_scope, BlockScalars* bs, int sms, cudaStream_t st);
// world scope: the ranks' [2][2048] 64-bit digit counts lie xstride floats apart in xall
void launch_global_decide(const float* xall, int xstride, int world, int side_mask, int pass, RowArrays ra, int Q, unsigned long long* hist,
                          uint32_t* cand, unsigned int cand_cap, BlockScalars* bs, cudaStream_t st);
// k nearest neighbours (npair_eval_knn): for each of the `rows` rows of the stored block S (stride ldS, a multiple of 32), query
// q0 + r, its k <= KNN_MAX_K largest columns j < ng other than column q0 + r + self_col0, by s descending (NaN last), then j ascending,
// into rows q0 + r of out_sim / out_idx [.. x k] (out_idx = col_base + j)
constexpr int KNN_MAX_K = 1024;
void launch_knn_select(const float* S, long long ldS, int rows, int ng, int k, int q0, int self_col0, int col_base, float* out_sim,
                       int* out_idx, cudaStream_t st);
// lets the current device launch the k-NN select with its dynamic shared memory (above the default limit)
cudaError_t allow_knn_select_smem();

// Retrieval evaluation (DESIGN 8; launchers in eval_kernels.cu).  `ra` holds only the per-query statistics of the similarity GEMM's
// EPI_STATS epilogue (st_*, cnt_same).
// max|x| over queries and gallery (g == NULL: the query set is the gallery) into the pre-zeroed *absmax_bits (NULL: no reduction),
// and the reset of the nq queries' statistics
void launch_eval_prep(const float* q, long long nq_el, const float* g, long long ng_el, unsigned int* absmax_bits, RowArrays ra, int nq,
                      int sms, cudaStream_t st);
// rows x D fp32 -> the A (side_b = 0) or B (side_b = 1) side of the similarity GEMM's operands (SimLayout), pre-scaled by
// pre_scale of `absmax` (>= 0) or of *absmax_bits; the side-A launch also stores the scale in bs
void launch_eval_split(const float* x, int rows, int D, long long Dp, int prec, int side_b, float absmax, const unsigned int* absmax_bits,
                       BlockScalars* bs, uint16_t* out, cudaStream_t st);
// best[i] = max same-label non-self similarity of query i, -inf when there is none
void launch_eval_best(RowArrays ra, int nq, float* best, cudaStream_t st);
// MAP@R (npair_eval_map_at_r).  seg[0..nq] = exclusive scan of R_i = cnt[i] (seg[nq] = sum R_i), and sum_err = {sum R_i, the error
// bits of bs}, whose bits it then clears
void launch_eval_seg_scan(const int* cnt, int nq, long long* seg, BlockScalars* bs, unsigned long long* sum_err, cudaStream_t st);
// dst = each query's segment of src sorted descending (ordered-uint keys, so the order is a total one and does not depend on src's)
void launch_eval_seg_sort(const int* cnt, const long long* seg, int nq, const float* src, float* dst, cudaStream_t st);
// MAP@R_i, R-Precision_i (NaN for R_i = 0 or a row whose gather count `fill` differs from R_i), optionally R_i and the best
// positive's rank, from the sorted positives and the bucket counts
void launch_eval_map_finish(const int* cnt, const long long* seg, const int* fill, const float* pos, const unsigned int* hist, int nq,
                            double* map_r, double* r_precision, int* R_out, int* rank, cudaStream_t st);
// k-means (npair_eval_kmeans, DESIGN 8.2).  sigma = pre_scale(max|x|).scale of the points, read from *absmax_bits.
// What each assignment sweep reports back to the host: assignments that changed, error bits, clusters that have a member
struct KmeansWords { unsigned int changed, err, nonempty, pad; };
constexpr int KM_INERTIA_BLOCKS = 256;          // fixed grid of the inertia reduction: its order does not depend on the device
// C[c] = x[rows[c]] (k x D)
void launch_km_gather(const float* x, int D, const int* rows, int k, float* C, cudaStream_t st);
// bias[c] = 0.5f * ||C_c||^2 in fp32; also zeroes counts[0..k) and *words
void launch_km_bias(const float* C, int k, int D, float* bias, int* counts, KmeansWords* words, cudaStream_t st);
// assign[i] = the column of the EPI_ARGMAX key best[i] (then zeroed); counts[a] += 1, words->changed / nonempty / err; accumulate:
// sums[a][d] += rint(x[i][d] * sigma * 2^32) in int64
void launch_km_assign(unsigned long long* best, const float* x, int n, int D, const unsigned int* absmax_bits, int k, int* assign,
                      int* counts, long long* sums, bool accumulate, KmeansWords* words, cudaStream_t st);
// C[c] = the fixed-point mean of cluster c where counts[c] > 0 (else unchanged); zeroes the sums
void launch_km_update(long long* sums, const int* counts, const unsigned int* absmax_bits, int k, int D, float* C, cudaStream_t st);
// *out = sum_i ||x_i - C[assign[i]]||^2 in fp64, in a fixed order (partial: KM_INERTIA_BLOCKS doubles of scratch)
void launch_km_inertia(const float* x, const float* C, const int* assign, int n, int D, double* partial, double* out, cudaStream_t st);
// k-means++ seeding (npair_eval_kmeans_seed, DESIGN 8.2): the points as int16 q = rint(x * sigma * 2^13), rows of KMS_DQ(D) elements,
// exact uint64 distances, one distance kernel and one update-and-sample kernel per step, blocks of KMS_THREADS points
constexpr int KMS_THREADS = 256;
constexpr int KMS_MAX_TRIALS = 255;             // u(seed, t, j) numbers j < 256 per step
__host__ __device__ inline long long kms_dq(long long D) { return (D + 15) / 16 * 16; }
// What the steps pass each other and the host: the potential phi, the error bits, the step's winning trial and the last-block tickets
struct KmSeedWords { unsigned long long phi; unsigned int err, jstar, ticket_dist, ticket_upd; };
// q = the points' int16 rows, norm[i] = sum q_i^2, dmin[i] = UINT64_MAX, cand[0] = step 0's row; DERR_KMEANS_NO_ARGMAX in
// words->err (pre-zeroed) for a non-finite x
void launch_kms_quantise(const float* x, int n, int D, const unsigned int* absmax_bits, unsigned long long seed, int16_t* q,
                         unsigned long long* norm, unsigned long long* dmin, int* cand, KmSeedWords* words, cudaStream_t st);
// Step t, its L trials cand[0, L): dist[j][i] = d(i, cand[j]), phi_j = sum_i min(dmin[i], dist[j][i]); the last block stores the
// trial of least phi_j (lowest j on ties) in words->jstar and its row in rows[t]
void launch_kms_distance(const int16_t* q, const unsigned long long* norm, const unsigned long long* dmin, int n, int D, const int* cand,
                         int L, int t, unsigned long long* dist, unsigned long long* phi_acc, int* rows, KmSeedWords* words, cudaStream_t st);
// dmin[i] = min(dmin[i], dist[jstar][i]); the last block scans the block totals into words->phi and, for L_next > 0, draws step t + 1's
// trials into cand[0, L_next)
void launch_kms_update(unsigned long long* dmin, const unsigned long long* dist, int n, unsigned long long seed, int t, int L_next,
                       unsigned long long* totals, unsigned long long* prefix, int* cand, KmSeedWords* words, cudaStream_t st);
// Hard negative class mining (npair_eval_class_batches, DESIGN 8.4): for each of the nb pools (pools [nb][P], P <= CLASS_POOL_MAX,
// distinct ids < the rows of S), the greedy batch of n >= 2 classes over the stored S (row c = class c, stride ldS) into batches
// [nb][n] and, unless NULL, the scores they were picked at into scores [nb][n] (NaN for the seed).  One block per batch, CB_ENTRIES
// pool positions per thread in registers, at most sms times the blocks an SM holds.
constexpr int CB_THREADS = 1024, CB_ENTRIES = 16;
constexpr int CLASS_POOL_MAX = 16384;
void launch_class_batches(const float* S, long long ldS, const int* pools, int P, int nb, int n, int* batches, float* scores, int sms,
                          cudaStream_t st);

}  // namespace npair
